"""Timing of the neuron-coverage arm (core/coverage_worker.py) and of KMNC's two CAM routes; not part of bench.py's
line.

    python tools/coverage_arm_bench.py [--steps K] [--warmup W] [--runs R] [--no-host]

Prints one JSON line with the card's name and power limit, read in the same call, and:
  * evaluate_all: `CoverageWorker` on a PyTorch copy of the MNIST case study's CNN (case_study_mnist.py:51-62, random
    weights, last bias shifted to balanced predictions as in tools/surprise_arm_bench.py) with the study's NC layers,
    Keras layers 0-3 = children [1, 2, 4, 5] (conv+ReLU, pool, conv+ReLU, pool: D = 21632 + 5408 + 7744 + 1600 =
    36384), 60 k training inputs, 10 k nominal and 10 k out-of-distribution inputs; per run (a fresh worker each) the
    training walk's wall time and per data set and metric the [setup, pred, quant, cam] seconds;
  * kmnc_routes: KMNC_2 on the nominal traces, the packed route (`KMNC.packed` + `cam_from_bits`) against the bucket
    route (`KMNC.buckets(device_out=True)` + `cam_from_buckets`), alternated call by call after W warm-up calls of
    each; median over K calls of the CUDA-event time around each whole route (the CAM loops' host syncs included) and
    of the wall time; the orders are asserted equal;
  * host_route: the reference's route for NAC_0.75 on the nominal traces — the dense profile `traces > 0.75` and
    `sum_score` in NumPy, then the NumPy greedy CAM (np_oracle.cam_oracle) — timed once and checked against the
    worker's order; `--no-host` reports it as not run.
Sizes computed from the shapes (not measured) are printed beside the timings.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from tools.quantifier_bench import card          # noqa: E402
from tools.surprise_arm_bench import balanced_model_and_inputs   # noqa: E402

NC_LAYERS = [1, 2, 4, 5]


def _rounded(times):
    return [round(float(t), 4) for t in times]


def evaluate_all_rows(worker_cls, model, train, datasets, runs):
    out = []
    for _ in range(runs):
        t0 = time.perf_counter()
        w = worker_cls(model, NC_LAYERS, train)
        run = {"training_walk_s": round(time.perf_counter() - t0, 3), "sets": {}}
        for ds, x in datasets.items():
            t0 = time.perf_counter()
            times, _, _ = w.evaluate_all(x, ds)
            run["sets"][ds] = {"wall_s": round(time.perf_counter() - t0, 3),
                               "times": {m: _rounded(t) for m, t in times.items()}}
        out.append(run)
    return out, w


def kmnc_route_rows(torch, w, flat, steps, warmup):
    from simple_tip_b200.core import prioritizers as P
    from simple_tip_b200.core.prioritizers import cam_from_bits, cam_from_buckets

    kmnc = w.metrics["KMNC_2"]
    scores = kmnc.packed(flat)[0].cpu().numpy().astype(np.int32)

    def packed():
        _, bits = kmnc.packed(flat)
        return list(cam_from_bits(scores, bits))

    def buckets():
        _, bucket = kmnc.buckets(flat, device_out=True)
        return list(cam_from_buckets(scores, bucket, kmnc.sections))
    assert packed() == buckets(), "KMNC_2 CAM orders of the two routes differ"
    routes = {"packed": packed, "buckets": buckets}
    for _ in range(warmup):
        for fn in routes.values():
            fn()
    dev_ms = {k: [] for k in routes}
    wall_ms = {k: [] for k in routes}
    for _ in range(steps):
        for name, fn in routes.items():           # alternated call by call
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.record()
            fn()
            b.record()
            b.synchronize()
            wall_ms[name].append((time.perf_counter() - t0) * 1e3)
            dev_ms[name].append(a.elapsed_time(b))
    row = {k: {"device_ms": round(float(np.median(dev_ms[k])), 3), "wall_ms": round(float(np.median(wall_ms[k])), 3)}
           for k in routes}
    packed()
    row["greedy_picks"] = int(P.LAST_GREEDY_PICKS)
    row["faster"] = min(routes, key=lambda k: row[k]["device_ms"])
    return row


def host_route_row(w, flat, nominal_order):
    from simple_tip_b200.core.neuron_coverage import sum_score
    from oracle import np_oracle

    host = flat.cpu().numpy()
    t0 = time.perf_counter()
    prof = host > 0.75                                  # neuron_coverage.py:58-62
    scores = sum_score(prof)
    t1 = time.perf_counter()
    order = np_oracle.cam_oracle(scores, prof)
    t2 = time.perf_counter()
    assert np.array_equal(order, nominal_order), "the host route's NAC_0.75 order differs from the worker's"
    return {"metric": "NAC_0.75", "quant_s": round(t1 - t0, 3), "cam_s": round(t2 - t1, 3),
            "dense_profile_mb": round(prof.nbytes / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--n-train", type=int, default=60_000)
    ap.add_argument("--n-test", type=int, default=10_000)
    ap.add_argument("--no-host", action="store_true", help="skip the reference's host route")
    args = ap.parse_args()

    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200.core.coverage_worker import CoverageWorker

    res = {"card": card()}
    model, train, datasets, hist = balanced_model_and_inputs(torch, args.n_train, args.n_test)
    n, d = args.n_test, 21632 + 5408 + 7744 + 1600
    words = int(_lib.load().tip_cover_packed_words(d))
    res["shapes"] = {"nc_layers": "children [1, 2, 4, 5] (Keras layers 0-3)", "d": d, "n_test": n,
                     "class_histogram": hist,
                     "test_traces_gb": round(n * d * 4 / 1e9, 2),
                     "kmnc2_bucket_ids_mb": round(n * d * 2 / 1e6, 1),
                     "kmnc2_bits_mb": round(n * 2 * words * 4 / 1e6, 1), "words_per_plane": words}
    runs, w = evaluate_all_rows(CoverageWorker, model, train, datasets, args.runs)
    res["evaluate_all"] = runs
    _, flat = w._traces(datasets["nominal"])
    res["kmnc_routes"] = kmnc_route_rows(torch, w, flat, args.steps, args.warmup)
    if args.no_host:
        res["host_route"] = "not run: --no-host"
    else:
        _, _, orders = w.evaluate_all(datasets["nominal"])
        res["host_route"] = host_route_row(w, flat, orders["NAC_0.75"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
