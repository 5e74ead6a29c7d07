"""Timing of pc-mlsa's setup on the device Gaussian-mixture backend (not part of bench.py's line).

    python tools/mlsa_bench.py [--steps K] [--warmup W] [--no-cpu]

Runs pc-mlsa's whole setup at the study's setting (handler_surprise.py:30-32: `MultiModalSA.build_by_class` with
`MLSA(x, num_components=3)` per predicted class) on C2's training shape, 60 k x 128 float32 rows in 10 classes,
plus one wide case, and prints one JSON line: the whole setup time and the per-class fits split into k-means init,
E-step pass (quadratic forms + responsibilities), M-step passes (moments + scatter), factorisation and the rest
(host syncs, launch gaps, the initial M-step); iterations per class; the passes' algorithmic fp64 rate
(4 N K D^2 flop per iteration, as sklearn computes it) against the H100 SXM data-sheet fp64 tensor rate; the
card's name and power limit; the sklearn fit on the host cores; and per class the largest relative difference
between score_samples of the device fit and of sklearn started from the same initial parameters.  Writes nothing
to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

FP64_TENSOR_PEAK = 67.0      # TFLOP/s, H100 SXM data sheet (700 W)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def synth(n, d, classes, seed):
    """ReLU-like activations of `classes` predicted classes: class-specific centres, a few dead units."""
    rng = np.random.default_rng(seed)
    y = rng.integers(0, classes, size=n)
    centres = rng.normal(size=(classes, d)).astype(np.float32)
    x = np.maximum(centres[y] + rng.normal(size=(n, d)).astype(np.float32), 0.0)
    x[:, : max(1, d // 32)] = 0.0
    return x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true", help="skip the sklearn host baseline and the parity block")
    args = ap.parse_args()

    import torch
    from sklearn.mixture import GaussianMixture as SkGM

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import MLSA, MultiModalSA

    dev = E.require_cuda()
    k = 3

    def setup_once(x, y):
        timing = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        MultiModalSA.build_by_class(x, y, lambda a, _: MLSA(a, num_components=k, backend="device"))
        torch.cuda.synchronize()
        whole = (time.perf_counter() - t0) * 1e3
        # the same per-class fits again, with CUDA events around the phases
        iters = []
        for c in np.unique(y):
            xc = E.to_device(x[y == c], dev)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                fit = E.gmm_fit(xc, k, timing=timing)
            iters.append((int(xc.shape[0]), fit["n_iter"]))
        return whole, timing, iters

    cases = []
    for name, n, d in (("C2 training shape", 60000, 128), ("wide", 60000, 1024)):
        x, y = synth(n, d, 10, seed=31)
        for _ in range(max(1, args.warmup)):
            setup_once(x, y)
        runs = [setup_once(x, y) for _ in range(max(1, args.steps))]
        whole = float(np.median([r[0] for r in runs]))
        timing = {key: float(np.median([r[1][key] for r in runs])) for key in runs[-1][1]}
        iters = runs[-1][2]
        flops = float(sum(4.0 * nc * k * d * d * it for nc, it in iters))
        passes_ms = timing["estep"] + timing["mstep"]
        case = {"workload": f"{name}: {n} x {d} float32 synthetic ReLU-like rows (seed 31), 10 classes, "
                            f"MultiModalSA.build_by_class with MLSA(num_components={k}, backend='device')",
                "setup_ms": whole, "iterations_per_class": [it for _, it in iters],
                "rows_per_class": [nc for nc, _ in iters],
                "split_ms_all_classes": {"kmeans_init": timing["kmeans"], "estep_passes": timing["estep"],
                                         "mstep_passes": timing["mstep"], "factorisation": timing["factor"],
                                         "other": timing["total"] - timing["kmeans"] - passes_ms - timing["factor"]},
                "fit_ms_all_classes": timing["total"],
                "passes_tflops": flops / (passes_ms * 1e-3) / 1e12,
                "passes_frac_of_fp64_tensor_peak": flops / (passes_ms * 1e-3) / 1e12 / FP64_TENSOR_PEAK,
                "rate_note": "algorithmic: 4*N*K*D^2 flop per EM iteration over the E-step + M-step pass time"}
        if not args.no_cpu and d <= 128:
            host_ms, parity = 0.0, {}
            for c in np.unique(y):
                xc = x[y == c]
                t0 = time.perf_counter()
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    SkGM(n_components=k).fit(xc)
                host_ms += (time.perf_counter() - t0) * 1e3
                m = MLSA(xc, num_components=k, backend="device")
                xd = E.to_device(xc, dev)
                w0, mu0, cov0, _, _, _ = E.gmm_init(xd, m.gmm.labels_init_, k, 1e-6)
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    sk = SkGM(k, weights_init=w0.cpu().numpy(), means_init=mu0.cpu().numpy(),
                              precisions_init=np.linalg.inv(cov0.cpu().numpy()), init_params="random",
                              random_state=0).fit(xc)
                ours, theirs = m.gmm.score_samples(xc), sk.score_samples(xc)
                parity[str(int(c))] = {"max_rel_diff": float(np.max(np.abs(ours - theirs) / np.abs(theirs))),
                                       "n_iter_device": m.gmm.n_iter_, "n_iter_sklearn": int(sk.n_iter_)}
            case["cpu_baseline"] = {"value_ms": host_ms, "cores": os.cpu_count(),
                                    "kind": "sklearn GaussianMixture(n_components=3).fit per class on the host"}
            case["parity_score_samples_vs_sklearn_same_init"] = parity
        cases.append(case)
    head = cases[0]
    line = {"metric": "pc_mlsa_setup_ms", "value": head["setup_ms"], "unit": "ms", "n_gpus": 1,
            "steps": max(1, args.steps), "warmup": max(1, args.warmup), "higher_is_better": False, "dtype": "f32",
            "data": "synthetic", "timing": "host clock around the synchronised setup; CUDA events per phase; "
                                           "median over steps", "card": card(),
            "fp64_tensor_peak_tflops": FP64_TENSOR_PEAK, "peak_source": "H100 SXM data sheet", "cases": cases}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
