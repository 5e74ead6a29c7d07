"""Timing of pc-mmdsa's k-means discriminator fit on the device backend (not part of bench.py's line).

    python tools/mmdsa_bench.py [--steps K] [--warmup W] [--no-cpu]

Runs the fit at the study's setting (handler_surprise.py:34-36: k = 2..5, n_init = 10, subsampling 0.3) on C2's
training shape, plus one wide case that shows the silhouette pass's tensor-core rate, and prints one JSON line:
device time per fit split into k-means (seeding + Lloyd + final relabel of all runs) and silhouette (sort + pack +
wgmma pass + finish), the silhouette's algorithmic TFLOP/s against the bf16 peak, the card's name and power limit,
the sklearn discriminator on the host cores, and the silhouette of sklearn's own labels computed both ways.
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
from bench import _peaks  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def synth(n, d, clusters, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(clusters, d)).astype(np.float32) * 3.0
    return centres[rng.integers(0, clusters, size=n)] + rng.normal(size=(n, d)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true", help="skip the sklearn host baseline and the parity block")
    args = ap.parse_args()

    import torch

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import _subsample_array

    dev = E.require_cuda()
    tflops_peak, _, peak_src = _peaks()
    potential_k, n_init = list(range(2, 6)), 10

    def fit_once(x):
        ev = lambda: torch.cuda.Event(enable_timing=True)
        km_ms = sil_ms = 0.0
        best = (-np.inf, None)
        for k in potential_k:
            e0, e1, e2 = ev(), ev(), ev()
            e0.record()
            _, labels, _, _ = E.kmeans_fit(x, k, n_init, 300, 1e-4, 0)
            e1.record()
            score = float(E.silhouette_samples(x, labels, k).mean())
            e2.record()
            torch.cuda.synchronize()
            km_ms += e0.elapsed_time(e1)
            sil_ms += e1.elapsed_time(e2)
            if score > best[0]:
                best = (score, k)
        return km_ms, sil_ms, best

    cases = []
    for name, n_full, d, sub in (("C2 training shape", 60000, 128, 0.3), ("wide", 64000, 2048, 1.0)):
        data = _subsample_array(sub, synth(n_full, d, 10, seed=21), seed=0)
        x = E.to_device(data, dev)
        n = x.shape[0]
        for _ in range(max(1, args.warmup)):
            fit_once(x)
        runs = [fit_once(x) for _ in range(max(1, args.steps))]
        km = float(np.median([r[0] for r in runs]))
        sil = float(np.median([r[1] for r in runs]))
        flops = float(n) * n * 2 * d * len(potential_k)
        case = {"workload": f"{name}: {n_full} x {d} float32 synthetic clusters (10 blobs, seed 21), subsampling {sub} "
                            f"-> {n} rows, k = {potential_k[0]}..{potential_k[-1]}, n_init = {n_init}",
                "fit_ms": km + sil, "kmeans_ms": km, "silhouette_ms": sil, "best_k": runs[-1][2][1],
                "best_silhouette": runs[-1][2][0],
                "silhouette_tflops": flops / (sil * 1e-3) / 1e12,
                "silhouette_tflops_note": "algorithmic: 2*d flops per (row, row) pair over the whole silhouette call "
                                          "(sort + pack + wgmma pass + finish); the split-bf16 operands carry 3 tensor "
                                          "products per algorithmic one",
                "silhouette_frac_of_peak": flops / (sil * 1e-3) / 1e12 / tflops_peak}
        if not args.no_cpu and d <= 128:
            from sklearn.cluster import KMeans
            from sklearn.metrics import silhouette_score

            from simple_tip_b200.core import clustering

            parity, host_best, host_ms, sk_sil_ms = {}, (-np.inf, None), 0.0, 0.0
            for k in potential_k:
                t0 = time.perf_counter()
                lab = KMeans(n_clusters=k, n_init=n_init, max_iter=300).fit_predict(data)
                t1 = time.perf_counter()
                sk = float(silhouette_score(data, lab))
                t2 = time.perf_counter()
                host_ms += (t2 - t0) * 1e3
                sk_sil_ms += (t2 - t1) * 1e3
                ours = clustering.silhouette_score(x, torch.from_numpy(lab).to(dev))
                parity[str(k)] = {"sklearn": sk, "ours": ours, "abs_diff": abs(sk - ours)}
                if sk > host_best[0]:
                    host_best = (sk, k)
            case["cpu_baseline"] = {"value_ms": host_ms, "silhouette_ms": sk_sil_ms, "cores": os.cpu_count(),
                                    "kind": "sklearn KMeans + silhouette_score on the host", "best_k": host_best[1]}
            case["parity_silhouette_of_sklearn_labels"] = parity
        cases.append(case)
        del x
    head = cases[0]
    line = {"metric": "mmdsa_discriminator_fit_ms", "value": head["fit_ms"], "unit": "ms", "n_gpus": 1,
            "steps": max(1, args.steps), "warmup": max(1, args.warmup), "higher_is_better": False, "dtype": "f32",
            "data": "synthetic", "timing": "CUDA events per k, median over steps", "card": card(),
            "peak_tflops": tflops_peak, "peak_source": peak_src, "cases": cases}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
