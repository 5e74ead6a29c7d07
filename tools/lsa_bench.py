"""Timing of pc-lsa's setup with LSA's device fit (not part of bench.py's line).

    python tools/lsa_bench.py [--steps K] [--warmup W] [--no-cpu]

Runs the setup at the study's setting (handler_surprise.py:26: `MultiModalSA.build_by_class` with `LSA(x)` per
predicted class, max_features 300) on 60 k float32 ReLU-like rows in 10 classes at the widths 128 (C2), 1600 (the
MNIST / Fashion-MNIST SA layer) and 2304 (CIFAR-10), and prints one JSON line: per width the device setup from
NumPy traces and from CUDA traces, the per-class fits split into the variance pass, the scatter, the factorisation
rounds, the whitening and the packing of the KDE operands (CUDA events and synchronised host clocks), the host fit
(`backend="host"`, the same setup with the reference's NumPy fit), the card's name and power limit, and a parity
block: per class `removed_neurons` and `prepare_failed` against the host fit and the largest relative score
difference against the host-fit LSA.  Writes nothing to the tree.
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
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true", help="skip the host-fit baseline and the parity block")
    args = ap.parse_args()
    warnings.simplefilter("ignore")

    import torch

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.stable_kde import StableGaussianKDE
    from simple_tip_b200.core.surprise import LSA, MultiModalSA

    dev = E.require_cuda()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    def device_lsa(a, _):
        return LSA(a, backend="device")

    def split(xd, yd):
        """per-class phases summed over the classes: variance pass, KDE fit phases, packing"""
        timing, var_ms, pack_ms = {}, 0.0, 0.0
        for c in np.unique(yd):
            xc = xd.index_select(0, torch.from_numpy(np.flatnonzero(yd == c)).to(dev))
            ms, (var, mean, _) = clock(lambda: E.col_var(xc))
            var_ms += ms
            cols = np.sort(np.argsort(var.cpu().numpy())[-min(300, xc.shape[1]):])
            fit = E.kde_fit(xc, cols, mean, timing=timing)
            if "p" in fit:                           # a failed fit (prepare_failed) has no operand to pack
                ms, _ = clock(lambda: E.KdeEngine(fit["p"]))
                pack_ms += ms
        return {"variance_pass": var_ms, "scatter": timing["scatter"], "factorisation_rounds": timing["factor"],
                "whitening": timing.get("whiten", 0.0), "kde_fit_total": timing["total"], "read_backs": timing["reads"],
                "packing": pack_ms}

    def once(x, y, xd):
        np_ms, _ = clock(lambda: MultiModalSA.build_by_class(x, y, device_lsa))
        cuda_ms, _ = clock(lambda: MultiModalSA.build_by_class(xd, y, device_lsa))
        return np_ms, cuda_ms, split(xd, y)

    cases = []
    for d in (128, 1600, 2304):
        x, y = synth(60000, d, 10, seed=41)
        xd = E.to_device(x, dev)
        for _ in range(max(1, args.warmup)):
            once(x, y, xd)
        runs = [once(x, y, xd) for _ in range(max(1, args.steps))]
        med = lambda i: float(np.median([r[i] for r in runs]))            # noqa: E731
        phases = {k: float(np.median([r[2][k] for r in runs])) for k in runs[-1][2]}
        case = {"workload": f"60000 x {d} float32 synthetic ReLU-like rows (seed 41), 10 classes, max_features 300",
                "pc_lsa_setup_device_from_numpy_ms": med(0), "pc_lsa_setup_device_from_cuda_ms": med(1),
                "per_class_phases_summed_ms": phases}
        if not args.no_cpu:
            host_ms, host = clock(lambda: MultiModalSA.build_by_class(x, y, lambda a, _: LSA(a)))
            devfit = MultiModalSA.build_by_class(xd, y, device_lsa)
            test, pred = x[::30], y[::30]
            parity = {}
            for c, sa in devfit.modal_sa.items():
                ref = host.modal_sa[c]
                rows = pred == c
                got, want = sa(test[rows]), ref(test[rows])
                f = np.isfinite(want) & np.isfinite(got)
                parity[str(int(c))] = {
                    "removed_neurons_equal": list(sa.removed_neurons) == list(ref.removed_neurons),
                    "prepare_failed_equal": sa.kde.prepare_failed == ref.kde.prepare_failed,
                    "same_infinite_scores": bool(np.array_equal(np.isinf(got), np.isinf(want))),
                    "max_rel_score_diff": float(np.max(np.abs(got[f] - want[f]) / np.abs(want[f]), initial=0.0))}
            host_fit_ms = 0.0
            for c in np.unique(y):
                xc = x[y == c]
                keep = np.argsort(np.var(xc, axis=0))[:-min(300, d)]
                t0 = time.perf_counter()
                kde = StableGaussianKDE.__new__(StableGaussianKDE)        # the host fit alone, no upload
                kde.dataset = np.delete(xc, keep, axis=1).T.astype(np.float64)
                kde.d, kde.n = kde.dataset.shape
                kde.weights = np.ones(kde.n) / kde.n
                kde.neff = 1.0 / np.sum(kde.weights ** 2)
                kde._compute_covariance()
                if not kde.prepare_failed:
                    _ = (kde.dataset.T - kde.dataset.mean(axis=1)) @ np.linalg.cholesky(kde.inv_cov)
                host_fit_ms += (time.perf_counter() - t0) * 1e3
            case["host_backend_setup_ms"] = host_ms
            case["host_fit_only_ms"] = {"value": host_fit_ms, "cores": os.cpu_count(),
                                        "kind": "np.cov + eigh rounds + inv + 2 cholesky + (x - mu) @ W per class, "
                                                "host float64, after the column selection"}
            case["parity_vs_host_fit"] = parity
        cases.append(case)
    line = {"metric": "pc_lsa_setup_device_from_numpy_ms", "value": cases[-1]["pc_lsa_setup_device_from_numpy_ms"],
            "unit": "ms", "n_gpus": 1, "steps": max(1, args.steps), "warmup": max(1, args.warmup),
            "higher_is_better": False, "dtype": "f32", "data": "synthetic",
            "timing": "host clock around the synchronised setup; CUDA events per fit phase; median over steps",
            "card": card(), "cases": cases}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
