"""What scoring the fault predictors of M case-study models in one stack costs against M single-model calls; not
part of bench.py.

    python tools/stacked_prio_bench.py [--models 1 8 32] [--cases mnist imdb] [--samplers head torch] [--rounds R]
                                       [--launches K] [--al-models 80]

Random-weight MNIST and IMDB case-study networks (seeded) on seeded synthetic inputs: MNIST 10 000 x 28 x 28 x 1
float32 (the study's test set), IMDB 2 500 x 100 int32 token ids (a tenth of the study's 25 000, as in
tools/mc_head_bench.py, so that M sequential torch-sampler calls stay within minutes).

1. The fault-predictor phase (point pass, the four softmax quantifiers and VR over 200 samples) per case study,
   sampler and M: `activations.get_pred_and_uncertainty_stack` on one stack of the M networks against M
   `get_pred_and_uncertainty` calls, one after the other.  After a warm-up of both paths, R rounds alternate the
   two; each wall time ends in a device synchronise.
2. `tip_mc_head_stack` on the M heads against M `tip_mc_head` launches on the same head inputs (10 000 MNIST rows,
   2 500 IMDB rows, 200 samples), by CUDA events around K repetitions of each; the outputs are compared bit for bit.
3. Active learning's evaluation of its retrained models: --al-models MNIST networks on the four splits of the study
   (10 k nominal + 10 k OOD inputs, observed share 0.5: four splits of 5 000), batch 128, stacked
   (`active_learning._evaluate_stack`) against one `_evaluate` per model, alternating R rounds; the accuracies of
   the two paths are compared.

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

SIZES = {"mnist": 10_000, "imdb": 2_500}


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, res


def networks(torch, name, m, seed):
    from simple_tip_b200.case_studies import imdb, mnist

    torch.manual_seed(seed)
    module = {"mnist": mnist, "imdb": imdb}[name]
    return [module.network().cuda().eval() for _ in range(m)]


def inputs(torch, name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "mnist":
        return torch.from_numpy(rng.random((n, 28, 28, 1), dtype=np.float32)).cuda()
    return torch.from_numpy(rng.integers(0, 2000, size=(n, 100)).astype(np.int32)).cuda()


def fault_predictors(torch, name, models_list, samplers, rounds):
    from simple_tip_b200.case_studies.stacked import stack
    from simple_tip_b200.core import activations as A

    x = inputs(torch, name, SIZES[name], 1)
    res = {}
    for sampler in samplers:
        warm = networks(torch, name, 2, 0)
        A.get_pred_and_uncertainty(warm[0], x[:500], sampler=sampler)
        A.get_pred_and_uncertainty_stack(stack(warm), x[:500], sampler=sampler)
        for m in models_list:
            models = networks(torch, name, m, m)
            net = stack(models).eval()
            seq, stk = [], []
            for _ in range(rounds):
                t, _ = timed(torch, lambda: A.get_pred_and_uncertainty_stack(net, x, sampler=sampler))
                stk.append(t)
                t, _ = timed(torch, lambda: [A.get_pred_and_uncertainty(mod, x, sampler=sampler) for mod in models])
                seq.append(t)
            res[f"{sampler}_M{m}"] = {"stacked_s": stk, "sequential_s": seq,
                                      "speedup_median": float(np.median(seq) / np.median(stk))}
            print(json.dumps({name: {f"{sampler}_M{m}": res[f"{sampler}_M{m}"]}}), file=sys.stderr, flush=True)
            del net, models
    return res


def head_kernel(torch, name, models_list, launches):
    from simple_tip_b200 import engine as E
    from simple_tip_b200.case_studies.stacked import stack
    from simple_tip_b200.core import activations as A

    x = inputs(torch, name, SIZES[name], 1)
    res = {}
    for m in models_list:
        net = stack(networks(torch, name, m, m)).eval()
        at, head = A.mc_head_layers_stack(net)
        trunk = []
        hook = list(net.children())[at].register_forward_pre_hook(lambda _m, inp: trunk.append(inp[0].detach()))
        with torch.no_grad():
            for s in range(0, x.shape[0], 500):
                net(net.stack_inputs([x[s:s + 500]] * m))
        hook.remove()
        h = torch.cat(trunk, dim=1).contiguous()
        layers = A._head_tensors(head, h.device)
        per_model = [[(k[i].contiguous(), b[i].contiguous(), p, act) for k, b, p, act in layers] for i in range(m)]
        seeds = list(range(m))
        # one launch of 200 samples over all rows of M models: bounded to ~2 GB of output
        rows = min(h.shape[1], max(1, (2 << 30) // (m * 200 * 4 * head[-1].module.kernel.shape[-1])))
        out = torch.empty((m, rows, 200, head[-1].module.kernel.shape[-1]), device="cuda")

        def stacked():
            E.mc_head_stack(h[:, :rows], layers, seeds, 200, out=out)

        def single():
            for i in range(m):
                E.mc_head(h[i, :rows], per_model[i], seeds[i], 200, out=out[i])

        stacked()
        want = out.clone()
        single()
        equal = bool(torch.equal(want, out))
        times = {}
        for label, fn in (("stacked", stacked), ("single", single), ("stacked2", stacked), ("single2", single)):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(launches):
                fn()
            end.record()
            torch.cuda.synchronize()
            times[label] = start.elapsed_time(end) / launches
        res[f"M{m}"] = {"rows": rows, "stacked_ms": [times["stacked"], times["stacked2"]],
                        "m_launches_ms": [times["single"], times["single2"]], "bit_equal": equal}
        del out, want, h
    return res


def al_evaluation(torch, m, rounds):
    from simple_tip_b200.core import active_learning as AL

    models = networks(torch, "mnist", m, 3)
    rng = np.random.default_rng(5)
    datasets = {}
    for ds in ("nominal", "ood"):
        for part in ("observed", "future"):
            datasets[ds, part] = (inputs(torch, "mnist", 5000, len(datasets)),
                                  torch.from_numpy(rng.integers(0, 10, 5000)).cuda())
    AL._evaluate_stack(models[:2], datasets, 10)
    AL._evaluate(models[0], datasets, 10)
    seq, stk = [], []
    for _ in range(rounds):
        t, got = timed(torch, lambda: AL._evaluate_stack(models, datasets, 10))
        stk.append(t)
        t, want = timed(torch, lambda: [AL._evaluate(mod, datasets, 10) for mod in models])
        seq.append(t)
    differing = sum(abs(a[k] - b[k]) > 0 for a, b in zip(got, want) for k in a)
    return {"models": m, "stacked_s": stk, "sequential_s": seq, "speedup_median": float(np.median(seq) / np.median(stk)),
            "accuracies_differing": int(differing), "max_abs_difference": max(abs(a[k] - b[k]) for a, b in
                                                                                zip(got, want) for k in a)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--cases", nargs="+", default=["mnist", "imdb"], choices=sorted(SIZES))
    ap.add_argument("--samplers", nargs="+", default=["head", "torch"], choices=["head", "torch"])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--al-models", type=int, default=80)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("stacked_prio_bench needs a CUDA device")
    res = {"card": card(), "rounds": args.rounds}
    for name in args.cases:
        res[name] = {"fault_predictors": fault_predictors(torch, name, args.models, args.samplers, args.rounds),
                     "mc_head_kernel": head_kernel(torch, name, args.models, args.launches)}
        print(json.dumps({name: res[name]["mc_head_kernel"]}), file=sys.stderr, flush=True)
    if args.al_models:
        res["active_learning_evaluation"] = al_evaluation(torch, args.al_models, args.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
