"""Where a test-prioritization run (core/prioritization.evaluate) spends its time; not part of bench.py's line.

    python tools/prioritization_bench.py [--backends device|default] [--n-train N] [--n-test N]

One `evaluate` call at the MNIST case study's settings on a PyTorch copy of its CNN (tools/quantifier_bench.mnist_cnn,
random weights, last bias shifted to balanced predictions as in tools/surprise_arm_bench.py), NC layers children
[1, 2, 4, 5] and SA layer children [5] as in tools/coverage_arm_bench.py and tools/surprise_arm_bench.py, 60 k
synthetic training inputs, 10 k nominal and 10 k out-of-distribution ones, labelled with the model's own predictions
of which a seeded 10 % are moved to another class (so both sets hold faults); every input stays in HBM.

Prints one JSON line with the card's name and power limit, read in the same call, and the wall time of each phase,
each ending in a device synchronise: the fault predictors per dataset (`get_pred_and_uncertainty`), the coverage
arm (the `CoverageWorker`'s construction and its two `evaluate_all`), the surprise arm (the `SurpriseHandler`'s
construction and its `evaluate_all`), writing the result files, and the APFDs; the whole call; and the peak of the
torch allocator over the call (`max_memory_allocated` / `max_memory_reserved`).  Then `results.write_apfd_table`
over the folder just written, and its time (pandas' first import timed apart).  The fits run with `B200TIP_{KDE,COV,GMM,KMEANS}=device` unless
`--backends default`.  A warm-up call on slices of the inputs comes first.  The result files go to a temporary
directory, removed afterwards; nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from tools.coverage_arm_bench import NC_LAYERS                        # noqa: E402
from tools.quantifier_bench import card                                # noqa: E402
from tools.surprise_arm_bench import DEVICE_BACKENDS, balanced_model_and_inputs   # noqa: E402

SA_LAYERS = [5]
PHASES = ("fp_nominal", "fp_ood", "coverage_arm", "surprise_arm", "files", "apfds")


def labelled(torch, model, x, rng, wrong=0.1):
    with torch.no_grad():
        y = torch.cat([model(x[i:i + 8192]).argmax(dim=1) for i in range(0, x.shape[0], 8192)]).cpu().numpy()
    flip = rng.random(y.size) < wrong
    y[flip] = (y[flip] + rng.integers(1, 10, int(flip.sum()))) % 10
    return torch.from_numpy(y).to(x.device)


def run(torch, model, data, out):
    """evaluate() with the arms, the result-file writers and the APFD helper wrapped in a synchronised wall clock."""
    from simple_tip_b200.core import activations, coverage_worker, prioritization, results, surprise_handler

    times = {name: 0.0 for name in PHASES}
    depth = [0]             # persist_tip writes through persist / persist_times: time the outermost call only

    def timed(name, fn):
        def call(*args, **kwargs):
            depth[0] += 1
            t0 = time.perf_counter()
            try:
                res = fn(*args, **kwargs)
                torch.cuda.synchronize()
            finally:
                depth[0] -= 1
            if depth[0] == 0:
                times[name() if callable(name) else name] += time.perf_counter() - t0
            return res
        return call

    fp_calls = []

    def fp_phase():
        fp_calls.append(1)
        return "fp_nominal" if len(fp_calls) == 1 else "fp_ood"

    class Worker(coverage_worker.CoverageWorker):
        __init__ = timed("coverage_arm", coverage_worker.CoverageWorker.__init__)
        evaluate_all = timed("coverage_arm", coverage_worker.CoverageWorker.evaluate_all)

    class Handler(surprise_handler.SurpriseHandler):
        __init__ = timed("surprise_arm", surprise_handler.SurpriseHandler.__init__)
        evaluate_all = timed("surprise_arm", surprise_handler.SurpriseHandler.evaluate_all)

    patches = [(activations, "get_pred_and_uncertainty", timed(fp_phase, activations.get_pred_and_uncertainty)),
               (coverage_worker, "CoverageWorker", Worker), (surprise_handler, "SurpriseHandler", Handler),
               (results, "apfd_values", timed("apfds", results.apfd_values))]
    patches += [(results, name, timed("files", getattr(results, name)))
                for name in ("persist", "persist_times", "persist_tip")]
    saved = [(mod, name, getattr(mod, name)) for mod, name, _ in patches]
    for mod, name, fn in patches:
        setattr(mod, name, fn)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        apfds = prioritization.evaluate(0, "mnist", model, nc_activation_layers=NC_LAYERS,
                                        sa_activation_layers=SA_LAYERS, output_folder=out, **data)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        for mod, name, fn in saved:
            setattr(mod, name, fn)
    return apfds, times, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backends", choices=["device", "default"], default="device")
    ap.add_argument("--n-train", type=int, default=60_000)
    ap.add_argument("--n-test", type=int, default=10_000)
    args = ap.parse_args()

    import torch

    from simple_tip_b200.core import results

    if args.backends == "device":
        os.environ.update(DEVICE_BACKENDS)
    else:
        for k in DEVICE_BACKENDS:
            os.environ.pop(k, None)
    res = {"card": card(), "settings": {"backends": args.backends, "n_train": args.n_train, "n_test": args.n_test,
                                        "nc_layers": NC_LAYERS, "sa_layers": SA_LAYERS, "batch_size": 128}}
    model, train, sets, hist = balanced_model_and_inputs(torch, args.n_train, args.n_test)
    rng = np.random.default_rng(0)
    data = {"training_dataset": train,
            "nominal_test_dataset": sets["nominal"], "nominal_test_labels": labelled(torch, model, sets["nominal"], rng),
            "ood_test_dataset": sets["ood"], "ood_test_labels": labelled(torch, model, sets["ood"], rng)}
    res["class_histogram"] = hist

    with tempfile.TemporaryDirectory() as tmp:
        # warm-up on slices (12 k training rows keep pc-lsa's per-class KDE covariance regular): cuDNN plans, the
        # library's modules, first-call allocations
        warm = {k: v[:12_000] if k.startswith("training") else v[:2000] for k, v in data.items()}
        np.random.seed(0)
        run(torch, model, warm, os.path.join(tmp, "warm"))

        out = os.path.join(tmp, "out")
        np.random.seed(0)
        torch.cuda.reset_peak_memory_stats()
        apfds, times, wall = run(torch, model, data, out)
        peak = {"allocated": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                "reserved": round(torch.cuda.max_memory_reserved() / 1e9, 2)}
        files = {d: len(os.listdir(os.path.join(out, d))) for d in ("priorities", "times")}
        t0 = time.perf_counter()
        import pandas  # noqa: F401   (write_apfd_table imports it on its first call; timed apart)
        pandas_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        results.write_apfd_table(out, ["mnist"])
        table_s = time.perf_counter() - t0
    res["phases_s"] = {name: round(t, 4) for name, t in times.items()}
    res["phases_s"]["rest"] = round(wall - sum(times.values()), 4)
    res["phases_s"]["wall"] = round(wall, 3)
    res["peak_gb"] = peak
    res["result_files"] = files
    res["apfd_table_s"] = {"pandas_import": round(pandas_s, 4), "write_apfd_table": round(table_s, 4)}
    res["apfd"] = {ds: {a: round(float(v), 4) for a, v in per_ds.items()} for ds, per_ds in apfds.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
