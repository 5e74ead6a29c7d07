"""What training M case-study models in one stack costs against M `fit` calls one after the other; not part of
bench.py.

    python tools/stacked_fit_bench.py [--models 1 8 80] [--cases mnist cifar10 imdb] [--rounds R] [--launches K] [--al]

Synthetic seeded inputs at the case studies' shapes: MNIST 60 000 x 28 x 28 x 1 float32 (batch 128), CIFAR-10
50 000 x 32 x 32 x 3 float64 as `load_datasets` gives it (batch 32), IMDB 25 000 x 100 int32 token ids (batch 32);
every model is trained on the whole pool with validation split 0.1.  Per case study and M, after a warm-up of both
paths, R rounds alternate one epoch of `core.training.fit_stack` over M fresh networks with M fresh networks
fitted one after the other by `core.training.fit`.  Each wall time ends in a device synchronise.  Per-step times are
wall time over the steps of the epoch (one stacked step takes all M models' batches).  Then the kernel times of
`tip_stack_gather` (inputs and targets of one step) and `tip_softmax_xent_seg` (the head of one step) at that M, by
CUDA events around K launches each.

--al: the retraining phase of one `active_learning.evaluate` at the MNIST case study's settings (60 k training,
10 k nominal + 10 k OOD inputs, observed share 0.5, 1000 selected, all `B200TIP_*=device`), one epoch per model,
sequential (`training_process` = `fit`) against stacked (`stacked_training_process` = `fit_stack`), timed around
the retraining calls only.  The result files go to a temporary directory.

Prints one JSON line with the card's name and power limit, read in the same call.  Nothing is written to the tree.
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

from tools.quantifier_bench import card                                   # noqa: E402

CASES = {"mnist": (60_000, 128), "cifar10": (50_000, 32), "imdb": (25_000, 32)}


def synced(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def pool(torch, name, n, seed=0):
    """Seeded synthetic inputs of the case study's shape and dtype and their one-hot labels, on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if name == "imdb":
        x = torch.randint(1, 2000, (n, 100), device="cuda", generator=g, dtype=torch.int32)
        x[:, :40] = 0
        classes = 2
    elif name == "cifar10":
        x, classes = torch.rand((n, 32, 32, 3), device="cuda", generator=g, dtype=torch.float64), 10
    else:
        x, classes = torch.rand((n, 28, 28, 1), device="cuda", generator=g), 10
    labels = torch.randint(0, classes, (n,), device="cuda", generator=g)
    return x, torch.nn.functional.one_hot(labels, classes).float()


def kernel_ms(torch, name, x, y, m, batch, launches):
    """CUDA-event times of one step's gathers and loss head for a stack of m models."""
    from simple_tip_b200 import engine as E
    from simple_tip_b200.case_studies import CASE_STUDIES, stacked

    n = x.shape[0]
    rows = torch.arange(n, device="cuda").expand(m, n).contiguous()
    perm = torch.stack([torch.randperm(n, device="cuda") for _ in range(m)])
    interleaved = stacked.stack([CASE_STUDIES[name].network()]).channels_interleaved
    xb = E.stack_gather(x, rows, perm, 0, batch, interleaved)
    yb = E.stack_gather(y, rows, perm, 0, batch)
    z = torch.randn(yb.shape, device="cuda")
    loss = torch.empty(m, device="cuda")
    correct = torch.empty(m, dtype=torch.int32, device="cuda")
    dz = torch.empty_like(z)

    def gather():
        E.stack_gather(x, rows, perm, batch, batch, interleaved, out=xb, check=False)
        E.stack_gather(y, rows, perm, batch, batch, out=yb, check=False)

    def time_it(fn):
        for _ in range(10):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        return round(a.elapsed_time(b) / launches, 4)
    return {"stack_gather_x_and_y_ms": time_it(gather),
            "softmax_xent_seg_ms": time_it(lambda: E.softmax_xent_seg(z, yb, loss, dz, correct)),
            "batch_bytes": xb.numel() * xb.element_size() + yb.numel() * yb.element_size()}


def run_case(torch, name, models, rounds, launches):
    from simple_tip_b200.case_studies import CASE_STUDIES
    from simple_tip_b200.core import training

    n, batch = CASES[name]
    network = CASE_STUDIES[name].network
    x, y = pool(torch, name, n)
    steps = -(-(n - training.validation_rows(n, 0.1)) // batch)

    def stack(m, rows_n=n):
        rows = torch.arange(rows_n, device="cuda").expand(m, rows_n).contiguous()
        return training.fit_stack([network().cuda() for _ in range(m)], x, y, rows, batch, 1)

    def sequential(m, rows_n=n):
        return [training.fit(network().cuda(), x[:rows_n], y[:rows_n], batch, 1) for _ in range(m)]

    synced(torch, lambda: stack(2, 6000))                 # warm-up: cuDNN plans, graph pools, library modules
    synced(torch, lambda: sequential(1, 6000))
    out = {"rows": n, "batch_size": batch, "steps_per_epoch": steps}
    for m in models:
        t_stack, t_seq = [], []
        for _ in range(rounds):
            trained, t = synced(torch, lambda: stack(m))
            t_stack.append(t)
            loss_stack = float(np.mean([mod.history["loss"][0] for mod in trained]))
            del trained
            trained, t = synced(torch, lambda: sequential(m))
            t_seq.append(t)
            loss_seq = float(np.mean([mod.history["loss"][0] for mod in trained]))
            del trained
            torch.cuda.empty_cache()
        out[f"M={m}"] = {
            "stacked_wall_s": [round(t, 3) for t in t_stack], "sequential_wall_s": [round(t, 3) for t in t_seq],
            "stacked_step_ms": [round(1e3 * t / steps, 4) for t in t_stack],
            "sequential_step_ms_per_model": [round(1e3 * t / (steps * m), 4) for t in t_seq],
            "speedup": round(min(t_seq) / min(t_stack), 3),
            "mean_epoch_loss": {"stacked": round(loss_stack, 4), "sequential": round(loss_seq, 4)},
            "kernels": kernel_ms(torch, name, x, y, m, batch, launches)}
    return out


def run_al(torch, out):
    from tools.active_learning_bench import labelled
    from tools.case_study_bench import blocks
    from tools.surprise_arm_bench import DEVICE_BACKENDS

    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import active_learning as AL
    from simple_tip_b200.core.training import fit, fit_stack

    os.environ.update(DEVICE_BACKENDS)
    x, lab = blocks(torch, 60_000, 1)
    model = fit(mnist.network().cuda(), x, torch.nn.functional.one_hot(lab, 10).float(), 128, 1, seed=0)
    nom, _ = blocks(torch, 10_000, 2)
    ood, _ = blocks(torch, 10_000, 3)
    ood = (1.0 - ood).contiguous()
    data = {"train_x": x, "train_y": labelled(torch, model, x), "nominal_test_x": nom,
            "nominal_test_labels": labelled(torch, model, nom), "ood_test_x": ood,
            "ood_test_labels": labelled(torch, model, ood)}
    retrain = []

    def training_process(xr, yr):
        m, t = synced(torch, lambda: fit(mnist.network().cuda(), xr, yr, 128, 1))
        retrain.append(t)
        return m

    def stacked_training_process(xp, yp, rows):
        ms, t = synced(torch, lambda: fit_stack([mnist.network().cuda() for _ in range(rows.shape[0])], xp, yp,
                                                rows, 128, 1))
        retrain.append(t)
        return ms

    res = {}
    for name, kw in (("sequential", {"training_process": training_process}),
                     ("stacked", {"training_process": None, "stacked_training_process": stacked_training_process})):
        retrain.clear()
        np.random.seed(0)
        (_, _, accs), wall = synced(torch, lambda: AL.evaluate(
            0, "mnist", model, nc_activation_layers=mnist.NC_ACTIVATION_LAYERS,
            sa_activation_layers=mnist.SA_ACTIVATION_LAYERS, observed_share=0.5, num_selected=1000, num_classes=10,
            output_folder=out, **data, **kw))
        res[name] = {"wall_s": round(wall, 2), "retraining_s": round(float(np.sum(retrain)), 2),
                     "retrained_models": len(accs),
                     "accuracy_retrained_mean": {f"{a}/{b}": round(float(np.mean([v[a, b] for v in accs.values()])), 4)
                                                 for a, b in next(iter(accs.values()))}}
    res["retraining_speedup"] = round(res["sequential"]["retraining_s"] / res["stacked"]["retraining_s"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", type=int, nargs="+", default=[1, 8, 80])
    ap.add_argument("--cases", nargs="+", default=list(CASES), choices=list(CASES))
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--al", action="store_true")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("stacked_fit_bench.py measures on a GPU; none is visible")
    res = {"card": card(), "settings": {"models": args.models, "rounds": args.rounds, "epochs": 1,
                                        "validation_split": 0.1, "tf32": torch.backends.cudnn.allow_tf32}}
    for name in args.cases:
        res[name] = run_case(torch, name, args.models, args.rounds, args.launches)
        print(json.dumps({name: res[name]}), file=sys.stderr, flush=True)
    if args.al:
        with tempfile.TemporaryDirectory() as out:
            res["active_learning"] = run_al(torch, out)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
