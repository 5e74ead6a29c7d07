"""Timing of the surprise-adequacy arm (core/surprise_handler.py, prioritizers.cam_from_surprise); not part of
bench.py's line.

    python tools/surprise_arm_bench.py [--steps K] [--backends default,device] [--skip NAME,...] [--no-sc-cam]

Prints one JSON line with the card's name and power limit and:
  * sc_cam: the SC-CAM order of N = 10 k and 100 k float64 scores with 1000 buckets, from NumPy and from CUDA scores:
    the one-pass path (`cam_from_surprise`) against the reference's route (the mapper's dense N x 1000 profile on the
    host, then `cam`: upload, bit-packing, greedy loop), median wall time of K calls each, with the greedy loop's own
    device time, the `tip_sc_cam` launches alone (CUDA events) and the shared `np.argsort` tail;
  * evaluate_all: `SurpriseHandler` on a PyTorch copy of the MNIST case study's CNN (case_study_mnist.py:51-62, random
    weights) with the SA layer the study uses (Keras layer 3, the second max-pool: 1600 wide), 60 k training inputs,
    10 k nominal and 10 k out-of-distribution inputs; per SA and data set the [setup, pred, sa, cam] seconds, once
    per backend set: "default" (the fits' default backends) and "device" (B200TIP_{KDE,COV,GMM,KMEANS}=device).
    Each SA runs in an `evaluate_all` call of its own after a warm-up call on slices of the inputs; a fit that
    raises is reported as such.  `--skip` leaves SAs out of the run (their rows then say "not measured"): sklearn's
    GaussianMixture on 1600-wide rows (pc-mlsa under the default backends) takes far longer than the other SAs.

Random weights predict a few classes for almost every input, which leaves classes too small for MLSA's 3 components,
for k-means up to k = 5, or with no training rows at all.  So the last layer's bias is shifted until the network
predicts every class about equally often on a pool of inputs (the weights stay random), and every set is drawn from
that pool's classes; the class histograms are printed.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from tools.quantifier_bench import card, device_ms, host_ms, mnist_cnn   # noqa: E402

DEVICE_BACKENDS = {"B200TIP_KDE": "device", "B200TIP_COV": "device", "B200TIP_GMM": "device",
                   "B200TIP_KMEANS": "device"}


def sc_cam_rows(steps, warmup):
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core import prioritizers as P
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    lib = _lib.load()
    rows = []
    for n in (10_000, 100_000):
        v = np.random.default_rng(n).gamma(2.0, size=n) * 10
        v_dev = torch.from_numpy(v).cuda()
        for src, x in (("numpy", v), ("cuda", v_dev)):
            def one_pass():
                ub = np.max(x) if src == "numpy" else x.max().item()
                return list(P.cam_from_surprise(x, SurpriseCoverageMapper(1000, ub)))

            def dense():
                h = x if src == "numpy" else x.cpu().numpy()
                return list(P.cam(h, SurpriseCoverageMapper(1000, np.max(h)).get_coverage_profile(h)))
            assert one_pass() == dense(), "SC-CAM orders differ"
            greedy = np.array(one_pass()[:P.LAST_GREEDY_PICKS], dtype=np.int64)
            one_ms = host_ms(one_pass, steps)
            dense_ms = host_ms(dense, steps)
            loop_ms = P.LAST_GREEDY_MS
            rows.append({"n": n, "scores": src, "picks": int(greedy.size), "one_pass_ms": round(one_ms, 3),
                         "dense_ms": round(dense_ms, 3), "dense_greedy_loop_ms": round(loop_ms, 3),
                         "dense_profile_mb": round(n * 1000 / 1e6, 1), "speedup": round(dense_ms / one_ms, 2)})
        mapper = SurpriseCoverageMapper(1000, np.max(v))
        t = torch.from_numpy(mapper.thresholds).cuda()
        first = torch.empty(1000, dtype=torch.int32, device="cuda")
        out = torch.empty(1001, dtype=torch.int32, device="cuda")

        def launch():
            _lib.check(lib.tip_sc_cam(E._p(v_dev), _lib.TIP_F64, n, E._p(t), 1000, E._p(first), E._p(out[1:]),
                                      E._p(out), E._stream()), "tip_sc_cam")
        kernel_us = device_ms(launch, steps * 5, warmup) * 1e3
        tail_ms = host_ms(lambda: list(P._tail_by_score(v.copy(), greedy)), steps)
        for r in rows[-2:]:
            r["tip_sc_cam_us"], r["argsort_tail_ms"] = round(kernel_us, 2), round(tail_ms, 3)
    return rows


def balanced_model_and_inputs(torch, n_train, n_test, pool_factor=2):
    """The CNN with its last bias shifted to balanced predictions, and (train, nominal, ood) inputs whose
    predicted classes all hold enough training rows."""
    model = mnist_cnn(torch).eval()
    rng = np.random.default_rng(0)

    def images(n):            # noise with a per-image contrast curve and brightness, so the features vary
        x = rng.random((n, 1, 28, 28)) ** rng.uniform(0.2, 5.0, (n, 1, 1, 1)) * rng.uniform(0.2, 1.0, (n, 1, 1, 1))
        return torch.from_numpy(x.astype(np.float32)).cuda()
    pool, ood = images(pool_factor * (n_train + n_test)), 1.0 - images(pool_factor * n_test)

    def batched(fn, x):
        with torch.no_grad():
            return torch.cat([fn(x[i:i + 8192]) for i in range(0, x.shape[0], 8192)])
    # the pre-softmax outputs vary little between inputs: shift the bias on them, the features do not depend on it
    z = batched(model[:-1], pool[:20_000]).double().cpu().numpy()
    bias, step = np.zeros(10), z.std(axis=0).mean()
    for it in range(500):
        freq = np.bincount((z + bias).argmax(axis=1), minlength=10) / z.shape[0]
        bias -= step * 2.0 * (freq - 0.1) * 0.99 ** it
    with torch.no_grad():
        model[-2].bias += torch.from_numpy(bias).float().cuda()
    p_pool = batched(lambda x: model(x).argmax(dim=1), pool).cpu().numpy()
    p_ood = batched(lambda x: model(x).argmax(dim=1), ood).cpu().numpy()
    counts = np.bincount(p_pool, minlength=10)
    classes = np.flatnonzero(counts >= (n_train + n_test) // 40)          # at least a quarter of a fair share
    keep = np.flatnonzero(np.isin(p_pool, classes))
    keep_ood = np.flatnonzero(np.isin(p_ood, classes))[:n_test]
    assert keep.size >= n_train + n_test and keep_ood.size == n_test, "too few inputs of the kept classes"
    train, nominal = pool[torch.from_numpy(keep[:n_train]).cuda()], pool[torch.from_numpy(keep[n_train:n_train + n_test]).cuda()]
    hist = {"train": np.bincount(p_pool[keep[:n_train]], minlength=10).tolist(),
            "nominal": np.bincount(p_pool[keep[n_train:n_train + n_test]], minlength=10).tolist(),
            "ood": np.bincount(p_ood[keep_ood], minlength=10).tolist()}
    return model, train, {"nominal": nominal, "ood": ood[torch.from_numpy(keep_ood).cuda()]}, hist


def evaluate_all_rows(torch, backends, skip, n_train, n_test):
    from simple_tip_b200.core.surprise_handler import SurpriseHandler

    model, train, datasets, hist = balanced_model_and_inputs(torch, n_train, n_test)
    out = {"class_histogram": hist, "sa_layer": "children index 5 (Keras layer 3), 1600 wide", "runs": {}}
    for name in backends:
        saved = {k: os.environ.get(k) for k in DEVICE_BACKENDS}
        if name == "device":
            os.environ.update(DEVICE_BACKENDS)
        else:
            for k in DEVICE_BACKENDS:
                os.environ.pop(k, None)
        try:
            h = SurpriseHandler(model, [5], train)
            run = {"train_ats_s": round(h.train_at_timer.get(), 4), "sa": {}}
            # one SA per evaluate_all call, so that a fit that raises costs only its own row
            for sa_name, fit in SurpriseHandler.TESTED_SA.items():
                if sa_name in skip:
                    run["sa"][sa_name] = "not measured"
                    continue
                h.TESTED_SA = {sa_name: fit}
                try:
                    # warm-up on slices (12 k training rows keep pc-lsa's per-class KDE covariance regular):
                    # cuDNN plans, the library's modules, first-call allocations
                    warm = SurpriseHandler(model, [5], train[:12_000])
                    warm.TESTED_SA = h.TESTED_SA
                    warm.evaluate_all({k: v[:2000] for k, v in datasets.items()})
                    np.random.seed(0)
                    t0 = time.perf_counter()
                    res = h.evaluate_all(datasets)[sa_name]
                except Exception as e:          # report and go on with the next SA
                    run["sa"][sa_name] = f"failed: {type(e).__name__}: {e}"
                    continue
                row = {ds: {"setup_s": round(t[0], 4), "pred_s": round(t[1], 4), "sa_s": round(t[2], 4),
                            "cam_s": round(t[3], 4), "max_score": float(np.max(s))} for ds, (s, _, t) in res.items()}
                row["wall_s"] = round(time.perf_counter() - t0, 3)
                run["sa"][sa_name] = row
            out["runs"][name] = run
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--backends", default="default,device")
    ap.add_argument("--skip", default="", help="comma-separated SA names to leave out of evaluate_all")
    ap.add_argument("--no-sc-cam", action="store_true")
    ap.add_argument("--n-train", type=int, default=60_000)
    ap.add_argument("--n-test", type=int, default=10_000)
    args = ap.parse_args()

    import torch

    res = {"card": card()}
    if not args.no_sc_cam:
        res["sc_cam"] = sc_cam_rows(args.steps, args.warmup)
    backends = [b for b in args.backends.split(",") if b]
    if backends:
        skip = {s for s in args.skip.split(",") if s}
        res["evaluate_all"] = evaluate_all_rows(torch, backends, skip, args.n_train, args.n_test)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
