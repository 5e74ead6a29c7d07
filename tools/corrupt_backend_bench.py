"""IMDB-C's corrupt() on the host and on the device, on text_corruptor_bench.py's synthetic 25 000-text x ~230-word
corpus (IMDB's test-set size): the wall time of corrupt(severity=0.5, seed=0) per backend, runs alternated, the
device's split into encode, census (kernel + the host's classification), kernels (CUDA events) and decode, and a
check that both backends return the same strings.  Prints one JSON line with the card's name and power limit.

    python tools/corrupt_backend_bench.py [--texts 25000] [--runs 2] [--out results/corrupt_backend_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from simple_tip_b200 import engine as E                      # noqa: E402
from simple_tip_b200.core import text_corruptor as T          # noqa: E402
from text_corruptor_bench import corpus, dictionary          # noqa: E402


def device_split(tc, texts):
    """One device corrupt() split into its stages (the same calls corrupt(backend="device") makes)."""
    timing = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    enc = [t.encode("utf-8") for t in texts]
    t1 = time.perf_counter()
    cdf = np.array([0.05, 0.35, 0.65, 1.0])
    out, bad = E.corrupt_texts(enc, tc.device_tables(), 0, 0.5, cdf, timing=timing)
    t2 = time.perf_counter()
    dec = [b.decode("utf-8", "surrogatepass") for b in out]
    t3 = time.perf_counter()
    assert bad is None
    return dec, {"encode_ms": round(1e3 * (t1 - t0), 1), "census_ms": round(timing["census_ms"], 1),
                 "kernels_ms": round(timing["kernels_ms"], 1), "device_call_ms": round(1e3 * (t2 - t1), 1),
                 "decode_ms": round(1e3 * (t3 - t2), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--texts", type=int, default=25000)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    E.require_cuda()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    texts = corpus(args.texts, dictionary(20000, seed=2))
    thesaurus = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden",
                             "text_corruptor_thesaurus.jsonl")
    res = {"card": card, "texts": len(texts), "bytes": sum(len(t.encode()) for t in texts)}
    with tempfile.TemporaryDirectory() as tmp:
        tc = T.TextCorruptor(texts, cache_dir=tmp, thesaurus_path=thesaurus)
        t0 = time.perf_counter()
        tc.device_tables()
        res["tables_s"] = round(time.perf_counter() - t0, 3)
        tc.corrupt(texts[:200], 0.5, 0, backend="device", force_recalculate=True)     # warm-up
        host_s, dev_s, outs = [], [], {}
        for _ in range(args.runs):                               # alternated
            for backend, times in (("host", host_s), ("device", dev_s)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[backend] = tc.corrupt(texts, 0.5, 0, backend=backend, force_recalculate=True)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
        dec, split = device_split(tc, texts)
    res.update({"host_corrupt_s": [round(t, 3) for t in host_s], "device_corrupt_s": [round(t, 3) for t in dev_s],
                "device_split": split, "equal": outs["host"] == outs["device"] == dec,
                "changed_texts": int(sum(a != b for a, b in zip(outs["device"], texts)))})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
