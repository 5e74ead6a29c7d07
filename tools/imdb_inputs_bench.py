"""The IMDB case study's inputs on the GPU: Tokenizer(num_words=2000).fit_on_texts on a training set and
texts_to_padded(maxlen=100) of a training and a test set, each 25 000 synthetic IMDB-like reviews of ~230 words
(Zipf over 60 000 words, capitals, punctuation, "<br />").

Reports, in one JSON line with the card's name and power limit:
  * wall times (median of --repeats after a warm-up) of fit_on_texts and of texts_to_padded per set, split into host
    encode (str -> UTF-8 bytes), device (upload, kernels, the fit's column download; ends in a synchronise) and
    building the dicts (word_counts, word_index, ...: the rest of fit_on_texts);
  * per-kernel device time from torch.profiler over one fit and one texts_to_padded, in a run of its own;
  * the host time of oracle/keras_text_oracle.py on the same texts: the Python restatement of keras_preprocessing
    1.1.2's loops, not Keras itself.

    python tools/imdb_inputs_bench.py [--texts 25000] [--repeats 3] [--out results/imdb_inputs_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import keras_text_oracle as K                   # noqa: E402
from simple_tip_b200 import engine as E                     # noqa: E402
from simple_tip_b200.core.tokenizer import Tokenizer        # noqa: E402


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def fit_phases(texts):
    """(encode s, device s, dicts s, total s) of one Tokenizer(num_words=2000).fit_on_texts(texts)."""
    tok = Tokenizer(num_words=2000)
    total, _ = _wall(lambda: tok.fit_on_texts(texts))
    enc, (raw, off) = _wall(lambda: E.encode_texts(texts, True))
    fresh = Tokenizer(num_words=2000)
    dev, _ = _wall(lambda: E.tok_fit(E.TokWords(raw, off, fresh._separators(), True, 64), fresh._device_vocab()))
    return enc, dev, total - enc - dev, total, tok


def pad_phases(tok, texts):
    total, out = _wall(lambda: tok.texts_to_padded(texts, 100))
    enc, (raw, off) = _wall(lambda: E.encode_texts(texts, True))

    def device():
        words = E.TokWords(raw, off, tok._separators(), True, 64)
        return E.tok_lookup(words, tok._device_vocab(), 2000, False, 100)[2].cpu()

    dev, _ = _wall(device)
    return enc, dev, total, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--texts", type=int, default=25000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    E.require_cuda()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    train = K.imdb_like_texts(args.texts, seed=1)
    test = K.imdb_like_texts(args.texts, seed=2)
    res = {"card": card, "texts": args.texts, "train_bytes": sum(len(t) for t in train),
           "train_words": sum(len(K.text_to_word_sequence(t)) for t in train[:1000]) * args.texts // 1000}

    fit_phases(train[:2000])                                        # warm-up: module load, allocator
    runs = [fit_phases(train) for _ in range(args.repeats)]
    med = lambda k: round(float(np.median([r[k] for r in runs])), 4)  # noqa: E731
    tok = runs[-1][4]
    res["fit_s"] = {"encode": med(0), "device": med(1), "dicts": med(2), "total": med(3),
                    "vocabulary": len(tok.word_counts)}
    res["padded_s"] = {}
    for name, texts in (("train", train), ("test", test)):
        pad_phases(tok, texts[:2000])
        runs = [pad_phases(tok, texts) for _ in range(args.repeats)]
        res["padded_s"][name] = {"encode": med(0), "device": med(1), "total": med(2)}

    # correctness at the timed size, and the restatement's host time
    t0 = time.perf_counter()
    ref = K.Tokenizer(num_words=2000)
    ref.fit_on_texts(train)
    t1 = time.perf_counter()
    seqs = {name: ref.texts_to_sequences(t) for name, t in (("train", train), ("test", test))}
    t2 = time.perf_counter()
    padded = {name: K.pad_sequences(s, maxlen=100) for name, s in seqs.items()}
    t3 = time.perf_counter()
    assert list(tok.word_counts.items()) == list(ref.word_counts.items()) and tok.word_index == ref.word_index
    for name, texts in (("train", train), ("test", test)):
        assert np.array_equal(tok.texts_to_padded(texts, 100), padded[name]), name
    res["restatement_host_s"] = {"fit": round(t1 - t0, 3), "sequences_per_set": round((t2 - t1) / 2, 3),
                                 "pad_per_set": round((t3 - t2) / 2, 3)}

    # per-kernel device time, profiler on (a run of its own)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        Tokenizer(num_words=2000).fit_on_texts(train)
        tok.texts_to_padded(test, 100)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if "tok_" in ev.key and "kernel" in ev.key:
            name = ev.key.split("(")[0].replace("void ", "").replace("tip::", "")
            kernels[name] = round(kernels.get(name, 0.0) + ev.device_time_total / 1e3, 3)
    res["kernel_ms"] = kernels
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
