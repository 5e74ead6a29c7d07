"""Timing of the uncertainty quantifiers (core/quantifiers.py, core/activations.get_pred_and_uncertainty); not part
of bench.py's line.

    python tools/quantifier_bench.py [--steps K] [--warmup W] [--e2e-n N] [--no-cpu]

Prints one JSON line with the card's name and power limit and:
  * point: MaxSoftmax, PCS, SoftmaxEntropy (and DeepGini beside them) on device-resident float32 softmax outputs at
    10 k x 10 (C1's shape), 1 M x 10 and 100 k x 1000: device time of one `tip_softmax_stat` launch by CUDA events
    (median of K), the bytes it must move (read p, write pred and the value) over that time, and that rate as a
    fraction of the H100 SXM's 3.35 TB/s; beside each the NumPy oracle on the host (median of K);
  * vr: VariationRatio from a dense 10 k x 200 x 10 float32 array: `tip_vote_add` alone (with its HBM rate), and
    the whole call (zeroing the counts, `tip_vote_add`, `tip_vote_finish`), the same way;
  * e2e: `get_pred_and_uncertainty` with S = 200 on a seeded PyTorch copy of the MNIST case study's CNN
    (case_study_mnist.py:51-62, random weights) over N synthetic 28 x 28 inputs: the wall time of the call and its
    own split — point forward pass, each point quantifier, MC-dropout forward passes, vote kernels.
Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM5 80 GB peak


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def device_ms(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def host_ms(fn, steps):
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def mnist_cnn(torch):
    """case_study_mnist.py:51-62 in PyTorch (Keras' Dense(10, softmax) -> Linear + Softmax)."""
    torch.manual_seed(0)
    return torch.nn.Sequential(
        torch.nn.Conv2d(1, 32, 3), torch.nn.ReLU(), torch.nn.MaxPool2d(2),
        torch.nn.Conv2d(32, 64, 3), torch.nn.ReLU(), torch.nn.MaxPool2d(2),
        torch.nn.Flatten(), torch.nn.Dropout(0.5), torch.nn.Linear(64 * 5 * 5, 10), torch.nn.Softmax(dim=1)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--e2e-n", type=int, default=10000)
    ap.add_argument("--no-cpu", action="store_true", help="skip the NumPy oracle on the host")
    args = ap.parse_args()

    import torch

    from oracle import np_oracle
    from oracle import quantifier_oracle as QO
    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.activations import get_pred_and_uncertainty
    from simple_tip_b200.core.quantifiers import Votes

    lib = _lib.load()
    dev = torch.device("cuda", 0)
    res = {"card": card(), "steps": args.steps, "point": [], "vr": None, "e2e": None}
    kinds = {"softmax": (_lib.STAT_MAX, QO.max_softmax), "pcs": (_lib.STAT_PCS, QO.pcs),
             "softmax_entropy": (_lib.STAT_ENTROPY, QO.softmax_entropy),
             "deep_gini": (_lib.STAT_GINI, np_oracle.deepgini_oracle)}
    for n, c in ((10_000, 10), (1_000_000, 10), (100_000, 1000)):
        p, _ = np_oracle.synth_softmax(n, c, seed=1)
        p_dev = torch.from_numpy(p).to(dev)
        pred = torch.empty(n, dtype=torch.int32, device=dev)
        out = torch.empty(n, dtype=torch.float32, device=dev)
        nbytes = n * c * 4 + n * 8
        for name, (kind, oracle) in kinds.items():
            def run():
                _lib.check(lib.tip_softmax_stat(E._p(p_dev), _lib.TIP_F32, n, c, kind, E._p(pred), E._p(out),
                                                E._stream()), "tip_softmax_stat")
            ms = device_ms(run, args.steps, args.warmup)
            row = {"quantifier": name, "n": n, "c": c, "device_us": round(ms * 1e3, 2),
                   "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                   "of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
            if not args.no_cpu:
                row["host_numpy_ms"] = round(host_ms(lambda: oracle(p), max(1, min(args.steps, 3))), 3)
            res["point"].append(row)
        del p_dev

    n, s, c = 10_000, 200, 10
    samples = np.random.default_rng(2).dirichlet(np.ones(c), size=(n, s)).astype(np.float32)
    s_dev = torch.from_numpy(samples).to(dev)

    pred_vr = torch.empty(n, dtype=torch.int32, device=dev)
    vr = torch.empty(n, dtype=torch.float64, device=dev)
    votes = Votes(n, c, dev)

    def run_add():          # the launch alone: Votes.add's argument checks would sit inside the timed window
        _lib.check(lib.tip_vote_add(E._p(s_dev), _lib.TIP_F32, n, c, s, c, s * c, E._p(votes.counts), E._stream()),
                   "tip_vote_add")

    def run_vr():
        v = Votes(n, c, dev)
        v.add(s_dev, s, sample_stride=c, row_stride=s * c)
        _lib.check(lib.tip_vote_finish(E._p(v.counts), n, c, s, E._p(pred_vr), E._p(vr), E._stream()),
                   "tip_vote_finish")
    add_ms = device_ms(run_add, args.steps, args.warmup)
    ms = device_ms(run_vr, args.steps, args.warmup)
    nbytes = n * s * c * 4
    res["vr"] = {"n": n, "samples": s, "c": c,
                 "vote_add_us": round(add_ms * 1e3, 2),
                 "vote_add_gb_per_s": round(nbytes / (add_ms * 1e-3) / 1e9, 1),
                 "vote_add_of_hbm_peak": round(nbytes / (add_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                 "device_us": round(ms * 1e3, 2),
                 "note": "device_us: zeroing the [n, c] counts + tip_vote_add + tip_vote_finish, launched from Python"}
    if not args.no_cpu:
        res["vr"]["host_numpy_ms"] = round(host_ms(lambda: QO.variation_ratio(samples), 3), 3)
    del s_dev

    model = mnist_cnn(torch)
    x = torch.from_numpy(np.random.default_rng(3).random((args.e2e_n, 1, 28, 28), dtype=np.float32)).to(dev)
    get_pred_and_uncertainty(model, x[:64], sample_size=200)            # warm-up: cuDNN plans, the library
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, unc, times = get_pred_and_uncertainty(model, x, sample_size=200, seed=0)
    wall = time.perf_counter() - t0
    res["e2e"] = {"n": args.e2e_n, "samples": 200, "batch_size": 32, "wall_s": round(wall, 3),
                  "point_forward_s": round(times["softmax"][1], 4),
                  "point_quantifiers_s": {k: round(v[2], 5) for k, v in times.items() if k != "VR"},
                  "mc_forward_s": round(times["VR"][1], 4), "vote_kernels_s": round(times["VR"][2], 4),
                  "mean_vr": round(float(np.mean(unc["VR"])), 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
