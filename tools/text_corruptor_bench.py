"""IMDB-C generation on the GPU: tip_levenshtein's time for the square dictionary matrix at V = 4 000 (the study's
dictionary_size), 16 000 and 50 000 (CUDA events, median of --repeats launches after a warm-up; word lengths drawn
like IMDB's common words, 5 to ~20 letters), with pairs/s; and the wall time of TextCorruptor's construction and of
corrupt(severity=0.5) on a synthetic 25 000-text x ~230-word corpus, IMDB's test-set size.  Prints one JSON line
with the card's name and power limit.

    python tools/text_corruptor_bench.py [--repeats 5] [--texts 25000] [--out results/text_corruptor_bench.json]
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
from simple_tip_b200 import engine as E                      # noqa: E402
from simple_tip_b200.core import text_corruptor as T          # noqa: E402

LETTERS = list("etaoinshrdlcumwfgypbvkjxqz")
FREQ = np.linspace(2.0, 0.1, len(LETTERS))
FREQ /= FREQ.sum()


def dictionary(v: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    words = set()
    while len(words) < v:
        k = int(np.clip(round(rng.gamma(6.0, 1.4)) + 5, 5, 30))
        words.add("".join(rng.choice(LETTERS, size=k, p=FREQ)))
    return sorted(words)


def kernel_ms(words, repeats: int) -> float:
    """Median CUDA-event time of the tip_levenshtein launch alone (host encoding and upload done once)."""
    from simple_tip_b200 import _lib

    ids, off = E.encode_words(words)
    dev = E.require_cuda()
    ids_d, off_d = torch.from_numpy(ids).to(dev), torch.from_numpy(off).to(dev)
    out = torch.empty((len(words), len(words)), dtype=torch.uint8, device=dev)
    lib, max_len = _lib.load(), int(np.max(np.diff(off)))

    def launch():
        _lib.check(lib.tip_levenshtein(E._p(ids_d), E._p(off_d), len(words), E._p(ids_d), E._p(off_d), len(words),
                                       max_len, 1, E._p(out), E._stream()), "tip_levenshtein")

    launch()
    torch.cuda.synchronize()
    assert torch.equal(out, E.levenshtein(words)), "the timed launch differs from engine.levenshtein"
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        launch()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def corpus(n_texts: int, vocab, seed: int = 1):
    rng = np.random.default_rng(seed)
    zipf = 1.0 / np.arange(1, len(vocab) + 1) ** 1.05
    zipf /= zipf.sum()
    short = ["a", "the", "of", "it", "is", "and", "to", ".", ",", "!"]
    texts = []
    for _ in range(n_texts):
        n = int(rng.integers(150, 310))
        picks = rng.choice(len(vocab), size=n, p=zipf)
        mask = rng.random(n) < 0.45
        texts.append(" ".join(short[k % len(short)] if m else vocab[k] for k, m in zip(picks, mask)))
    return texts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--texts", type=int, default=25000)
    ap.add_argument("--sizes", default="4000,16000,50000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    E.require_cuda()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"card": card, "kernel": []}
    for v in map(int, args.sizes.split(",")):
        words = dictionary(v)
        ms = kernel_ms(words, args.repeats)
        res["kernel"].append({"V": v, "ms": round(ms, 3), "pairs_per_s": v * v / (ms * 1e-3)})
        print(json.dumps(res["kernel"][-1]), flush=True)

    vocab = dictionary(20000, seed=2)
    texts = corpus(args.texts, vocab)
    thesaurus = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden",
                             "text_corruptor_thesaurus.jsonl")
    with tempfile.TemporaryDirectory() as tmp:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tc = T.TextCorruptor(texts, cache_dir=tmp, thesaurus_path=thesaurus)
        t1 = time.perf_counter()
        out = tc.corrupt(texts, severity=0.5, seed=0)
        t2 = time.perf_counter()
    res["corruptor"] = {"texts": len(texts), "words": int(sum(len(t.split()) for t in texts)),
                        "dictionary": len(tc.common_words), "construct_s": round(t1 - t0, 3),
                        "corrupt_s": round(t2 - t1, 3), "changed_texts": int(sum(a != b for a, b in zip(out, texts)))}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
