"""What running the coverage arm of M case-study models as one stack costs against M single-model arms; not part of
bench.py.

    python tools/stacked_coverage_bench.py [--models 1 8 16] [--cases mnist imdb] [--rounds R] [--launches K]

Random-weight MNIST and IMDB case-study networks (seeded) on seeded synthetic inputs: MNIST 60 000 training and two
test sets of 10 000 x 28 x 28 x 1 float32 (the study's sizes), IMDB 25 000 training and two test sets of 10 000 x 100
int32 token ids.  Badges of 128, as the study's prioritization run.

1. The whole arm per case study and M: one `StackedCoverageWorker` on a stack of the M networks (training walk, then
   `evaluate_all` on both test sets) against M `CoverageWorker`s doing the same one after the other.  After a warm-up
   of both paths, R rounds alternate the two; each wall time ends in a device synchronise.  The torch allocator's
   peak is recorded per path (reset before each timed run).
2. The greedy CAM kernel alone on the M models' KMNC_2 profiles of the first test set (the stack's own traces):
   one `tip_cam_bits_stack` launch against M `tip_cam_bits` launches, each with gains initialised in the call and
   enough rounds to finish in one launch, by CUDA events around K repetitions; the orders and states are compared.

Prints one JSON line with the card's name and power limit, read in the same call.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from tools.quantifier_bench import card                                   # noqa: E402

TRAIN = {"mnist": 60_000, "imdb": 25_000}
TEST = 10_000
BATCH = 128


def timed(torch, fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated(), res


def networks(torch, name, m, seed):
    from simple_tip_b200.case_studies import imdb, mnist

    torch.manual_seed(seed)
    module = {"mnist": mnist, "imdb": imdb}[name]
    return [module.network().cuda().eval() for _ in range(m)], module.NC_ACTIVATION_LAYERS


def inputs(torch, name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "mnist":
        return torch.from_numpy(rng.random((n, 28, 28, 1), dtype=np.float32)).cuda()
    return torch.from_numpy(rng.integers(0, 2000, size=(n, 100)).astype(np.int32)).cuda()


def stacked_arm(net, layers, x_train, tests):
    from simple_tip_b200.core.coverage_worker import StackedCoverageWorker

    worker = StackedCoverageWorker(net, layers, x_train, batch_size=BATCH)
    return [worker.evaluate_all(x) for x in tests]


def sequential_arm(models, layers, x_train, tests):
    from simple_tip_b200.core.coverage_worker import CoverageWorker

    out = []
    for model in models:
        worker = CoverageWorker(model, layers, x_train, batch_size=BATCH)
        out.append([worker.evaluate_all(x) for x in tests])
        del worker
    return out


def whole_arm(torch, name, models_list, rounds):
    from simple_tip_b200.case_studies.stacked import stack

    x_train = inputs(torch, name, TRAIN[name], 1)
    tests = [inputs(torch, name, TEST, 2), inputs(torch, name, TEST, 3)]
    warm, layers = networks(torch, name, 2, 0)
    stacked_arm(stack(warm), layers, x_train[:1000], [t[:1000] for t in tests])
    sequential_arm(warm[:1], layers, x_train[:1000], [t[:1000] for t in tests])
    res = {}
    for m in models_list:
        models, layers = networks(torch, name, m, m)
        net = stack(models).eval()
        seq, stk, seq_peak, stk_peak = [], [], 0, 0
        for _ in range(rounds):
            t, peak, _ = timed(torch, lambda: stacked_arm(net, layers, x_train, tests))
            stk.append(t)
            stk_peak = max(stk_peak, peak)
            t, peak, _ = timed(torch, lambda: sequential_arm(models, layers, x_train, tests))
            seq.append(t)
            seq_peak = max(seq_peak, peak)
        res[f"M{m}"] = {"stacked_s": stk, "sequential_s": seq, "speedup_median": float(np.median(seq) / np.median(stk)),
                        "stacked_peak_gb": stk_peak / 1e9, "sequential_peak_gb": seq_peak / 1e9}
        print(json.dumps({name: {f"M{m}": res[f"M{m}"]}}), file=sys.stderr, flush=True)
        del net, models
    return res


def cam_kernel(torch, name, models_list, launches):
    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E
    from simple_tip_b200.case_studies.stacked import stack
    from simple_tip_b200.core.coverage_worker import StackedCoverageWorker

    lib = _lib.load()
    x_train = inputs(torch, name, TRAIN[name], 1)
    x_test = inputs(torch, name, TEST, 2)
    res = {}
    for m in models_list:
        models, layers = networks(torch, name, m, m)
        worker = StackedCoverageWorker(stack(models).eval(), layers, x_train, batch_size=BATCH)
        flat, _ = worker._traces(x_test)
        kmnc = worker.metrics["KMNC_2"]
        bits = torch.stack([kmnc[k].packed(flat[k])[1] for k in range(m)]).contiguous()
        del flat, worker
        n, words = int(bits.shape[1]), int(bits.shape[2])
        rounds = (n + 2) & ~1                           # one launch runs every greedy round
        cand = torch.zeros(4 * _lib.CAM_MAX_BLOCKS, dtype=torch.int32, device="cuda")
        buf = {k: (torch.empty((m, n), dtype=torch.int32, device="cuda"),
                   torch.zeros((m, 2 * words), dtype=torch.int32, device="cuda"),
                   torch.zeros((m, n), dtype=torch.int32, device="cuda"),
                   torch.zeros((m, 4), dtype=torch.int32, device="cuda")) for k in ("stack", "single")}

        def reset(k):
            for t in buf[k][1:]:
                t.zero_()

        def stacked():
            gain, covered, order, state = buf["stack"]
            _lib.check(lib.tip_cam_bits_stack(E._p(bits), m, n, words, E._p(gain), E._p(covered), E._p(cand),
                                              E._p(order), E._p(state), rounds, 1, E._stream()), "tip_cam_bits_stack")

        def single():
            gain, covered, order, state = buf["single"]
            for k in range(m):
                _lib.check(lib.tip_cam_bits(E._p(bits[k]), n, words, E._p(gain[k]), E._p(covered[k]), E._p(cand),
                                            E._p(order[k]), E._p(state[k]), rounds, 1, E._stream()), "tip_cam_bits")

        times = {"stacked": [], "single": []}
        for label, fn in (("stacked", stacked), ("single", single)) * 2:
            total = 0.0
            for _ in range(launches):
                reset(label if label == "single" else "stack")
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                fn()
                end.record()
                torch.cuda.synchronize()
                total += start.elapsed_time(end)
            times[label].append(total / launches)
        st_s, st_1 = buf["stack"][3].cpu().numpy(), buf["single"][3].cpu().numpy()
        equal = bool(np.array_equal(st_s, st_1) and torch.equal(buf["stack"][2], buf["single"][2]))
        res[f"M{m}"] = {"n": n, "words": words, "picks": st_s[:, 0].tolist(), "stacked_ms": times["stacked"],
                        "m_launches_ms": times["single"], "orders_equal": equal}
        print(json.dumps({name: {f"kernel_M{m}": res[f"M{m}"]}}), file=sys.stderr, flush=True)
        del bits, buf
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", type=int, nargs="+", default=[1, 8, 16])
    ap.add_argument("--cases", nargs="+", default=["mnist", "imdb"], choices=sorted(TRAIN))
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--launches", type=int, default=3)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("stacked_coverage_bench needs a CUDA device")
    res = {"card": card(), "rounds": args.rounds, "train": TRAIN, "test": [TEST, TEST], "batch": BATCH}
    for name in args.cases:
        res[name] = {"whole_arm": whole_arm(torch, name, args.models, args.rounds),
                     "cam_kernel_kmnc2": cam_kernel(torch, name, args.models, args.launches)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
