"""Timing of pc-mdsa's and pc-mmdsa's setup on the device EmpiricalCovariance backend (not part of bench.py's line).

    python tools/mdsa_bench.py [--steps K] [--warmup W] [--no-cpu]

Runs the setups at the study's settings (handler_surprise.py:28 and :34-36: `MultiModalSA.build_by_class` with
`MDSA(x)` per predicted class; `build_with_kmeans` with k = 2..5 and subsampling 0.3, here on the device k-means)
on 60 k float32 ReLU-like rows in 10 classes at the widths 128 (C2), 1600 (the MNIST / Fashion-MNIST SA layer) and
2304 (CIFAR-10), and prints one JSON line: per width the whole setup times, the per-class fits split into
cov_location, scatter and eigh (CUDA events), the host-to-device upload of the class rows, the card's name and power
limit, sklearn's `EmpiricalCovariance().fit` per class on the host cores, and a parity block: per class the rank
against scipy's pinvh and the largest relative difference of `mahalanobis` against sklearn.  Writes nothing to
the tree.
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
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true", help="skip the sklearn host baseline and the parity block")
    args = ap.parse_args()

    import torch
    from scipy import linalg
    from sklearn.covariance import EmpiricalCovariance as SkEC

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import MDSA, MultiModalSA

    dev = E.require_cuda()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    def once(x, y):
        pc_ms, _ = clock(lambda: MultiModalSA.build_by_class(x, y, lambda a, _: MDSA(a, backend="device")))
        mm_ms, mm = clock(lambda: MultiModalSA.build_with_kmeans(
            x, y, lambda a, _: MDSA(a, backend="device"), potential_k=range(2, 6), subsampling=0.3,
            backend="device"))
        timing, upload = {}, 0.0
        for c in np.unique(y):
            ms, xc = clock(lambda: E.to_device(x[y == c], dev))
            upload += ms
            E.cov_fit(xc, timing=timing)
        return pc_ms, mm_ms, timing, upload, len(mm.modal_sa)

    cases = []
    for d in (128, 1600, 2304):
        x, y = synth(60000, d, 10, seed=41)
        for _ in range(max(1, args.warmup)):
            once(x, y)
        runs = [once(x, y) for _ in range(max(1, args.steps))]
        med = lambda i: float(np.median([r[i] for r in runs]))
        timing = {k: float(np.median([r[2][k] for r in runs])) for k in runs[-1][2]}
        case = {"workload": f"60000 x {d} float32 synthetic ReLU-like rows (seed 41), 10 classes",
                "pc_mdsa_setup_ms": med(0), "pc_mmdsa_setup_ms": med(1), "pc_mmdsa_modals": runs[-1][4],
                "per_class_fits_ms": {"cov_location": timing["cov_location"], "scatter": timing["scatter"],
                                      "eigh": timing["eigh"], "total": timing["total"]},
                "class_rows_upload_ms": med(3)}
        if not args.no_cpu:
            host_ms, parity = 0.0, {}
            test = x[::30]
            for c in np.unique(y):
                xc = x[y == c]
                t0 = time.perf_counter()
                sk = SkEC().fit(xc)
                host_ms += (time.perf_counter() - t0) * 1e3
                m = MDSA(xc, backend="device")
                s = linalg.eigvalsh(sk.covariance_)
                cut = d * np.finfo(np.float64).eps * np.max(np.abs(s))
                want = sk.mahalanobis(test)
                parity[str(int(c))] = {"rank_device": m.covariance_matrix.rank_,
                                       "rank_scipy": int(np.sum(np.abs(s) > cut)),
                                       "mahalanobis_max_rel_diff": float(np.max(np.abs(m(test) - want) / np.abs(want)))}
            case["cpu_baseline"] = {"value_ms": host_ms, "cores": os.cpu_count(),
                                    "kind": "sklearn EmpiricalCovariance().fit per class on the host"}
            case["parity_vs_sklearn"] = parity
        cases.append(case)
    line = {"metric": "pc_mdsa_setup_ms", "value": cases[-1]["pc_mdsa_setup_ms"], "unit": "ms", "n_gpus": 1,
            "steps": max(1, args.steps), "warmup": max(1, args.warmup), "higher_is_better": False, "dtype": "f32",
            "data": "synthetic", "timing": "host clock around the synchronised setup; CUDA events per phase; "
                                           "median over steps", "card": card(), "cases": cases}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
