"""What one case-study training costs: the graph-captured `fit` against the eager torch loop; not part of bench.py.

    python tools/case_study_bench.py [--epochs E] [--rounds R] [--adam-launches K] [--al]

One MNIST case-study model trained with its recipe (batch 128, validation split 0.1) on 60 k synthetic inputs
(54 000 trained rows, 422 steps per epoch), two ways, alternated R times after a warm-up of both:
* `core.training.fit` on `case_studies.mnist.network()` (NHWC inputs, Keras' Adam, CUDA graphs);
* the eager loop of `tools/active_learning_bench.make_training_process` (torch's Adam, NLL of the clamped log of
  the softmax output, all 60 k rows: 469 steps per epoch) on the same inputs viewed NCHW.
Each wall time ends in a device synchronise.  Then the kernel time of `tip_keras_adam` against
`torch.optim.Adam(foreach=True)` over the same network's parameters, by CUDA events around K launches each.

--al: one `active_learning.evaluate` at the MNIST case study's settings (60 k training, 10 k nominal + 10 k OOD
inputs, observed share 0.5, 1000 selected, layers [0, 1, 2, 3] / [3], all `B200TIP_*=device`) with the case study's
`fit` for 1 epoch as `training_process`; the original model is a case-study network fitted for one epoch on a
learnable synthetic task (the class is the bright 7 x 7 block), labels = its predictions.  The result files go to a
temporary directory.

Prints one JSON line with the card's name and power limit, read in the same call.  Inputs are synthetic (seeded);
nothing is written to the tree.
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

from tools.active_learning_bench import labelled, make_training_process   # noqa: E402
from tools.quantifier_bench import card                                   # noqa: E402
from tools.surprise_arm_bench import DEVICE_BACKENDS                      # noqa: E402


def blocks(torch, n, seed):
    """n NHWC [28, 28, 1] float32 images whose class is the bright 7 x 7 block of a 4 x 4 grid, on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    labels = torch.randint(0, 10, (n,), device="cuda", generator=g)
    x = torch.rand((n, 28, 28), device="cuda", generator=g) * 0.35
    r, k = labels // 4, labels % 4
    rows = torch.arange(28, device="cuda")
    mask = ((rows[None, :] // 7) == r[:, None])[:, :, None] & ((rows[None, :] // 7) == k[:, None])[:, None, :]
    return (x + 0.6 * mask).unsqueeze(-1).contiguous(), labels


def synced(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def adam_kernel_ms(torch, launches):
    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core.training import KerasAdam

    net = mnist.network().cuda()
    params = list(net.parameters())
    grads = [torch.randn_like(p) * 1e-2 for p in params]
    opt = KerasAdam(params)
    table = opt.table(grads)
    ref = [p.detach().clone().requires_grad_(True) for p in params]
    for p, g in zip(ref, grads):
        p.grad = g.clone()
    torch_opt = torch.optim.Adam(ref, foreach=True)

    def time_it(step):
        for _ in range(10):
            step()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(launches):
            step()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / launches

    res = {}
    for name, step in (("tip_keras_adam", lambda: opt.step(table)), ("torch_adam_foreach", torch_opt.step)) * 2:
        res.setdefault(name, []).append(round(time_it(step), 4))
    res["parameters"] = sum(p.numel() for p in params)
    res["tensors"] = len(params)
    return res


def run_al(torch, out):
    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import active_learning as AL
    from simple_tip_b200.core.training import fit

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

    def call(d, k):
        return AL.evaluate(0, "mnist", model, nc_activation_layers=mnist.NC_ACTIVATION_LAYERS,
                           sa_activation_layers=mnist.SA_ACTIVATION_LAYERS, training_process=training_process,
                           observed_share=0.5, num_selected=k, num_classes=10, output_folder=out, **d)

    np.random.seed(0)
    warm = {k: v[:12_000] if k.startswith("train") else v[:2000] for k, v in data.items()}
    call(warm, 100)
    retrain.clear()
    np.random.seed(0)
    (orig, _, accs), wall = synced(torch, lambda: call(data, 1000))
    r = np.array(retrain)
    return {"wall_s": round(wall, 2), "retraining_total_s": round(float(r.sum()), 2), "models": int(r.size),
            "retraining_per_model_s": {"min": round(float(r.min()), 3), "median": round(float(np.median(r)), 3),
                                       "max": round(float(r.max()), 3)},
            "retraining_share": round(float(r.sum()) / wall, 3),
            "accuracy_original": {f"{a}/{b}": v for (a, b), v in orig.items()},
            "accuracy_retrained_mean": {f"{a}/{b}": round(float(np.mean([v[a, b] for v in accs.values()])), 4)
                                        for a, b in orig}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=15)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--adam-launches", type=int, default=500)
    ap.add_argument("--al", action="store_true")
    args = ap.parse_args()

    import torch

    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import active_learning, training

    if not torch.cuda.is_available():
        raise SystemExit("case_study_bench.py measures on a GPU; none is visible")
    res = {"card": card(), "settings": {"epochs": args.epochs, "rounds": args.rounds, "rows": 60_000,
                                        "batch_size": 128, "validation_split": 0.1}}
    x, lab = blocks(torch, 60_000, 0)
    y = torch.nn.functional.one_hot(lab, 10).float()
    x_nchw = x.permute(0, 3, 1, 2)
    steps_fit = -(-(60_000 - training.validation_rows(60_000, 0.1)) // 128)
    steps_eager = -(-60_000 // 128)

    def run_fit(epochs, n=60_000):
        return training.fit(mnist.network().cuda(), x[:n], y[:n], 128, epochs)

    def run_eager(epochs, n=60_000):
        return make_training_process(torch, epochs)(x_nchw[:n], y[:n])

    synced(torch, lambda: run_fit(1, 6000))                 # warm-up: cuDNN plans, graph pools, library modules
    synced(torch, lambda: run_eager(1, 6000))
    times = {"fit": [], "eager": []}
    hx, hl = blocks(torch, 10_000, 9)
    acc = {}
    for _ in range(args.rounds):
        m, t = synced(torch, lambda: run_fit(args.epochs))
        times["fit"].append(t)
        acc["fit"] = active_learning.accuracy(m, hx, hl)
        m, t = synced(torch, lambda: run_eager(args.epochs))
        times["eager"].append(t)
        acc["eager"] = active_learning.accuracy(m, hx.permute(0, 3, 1, 2), hl)
    res["training"] = {
        name: {"wall_s": [round(t, 3) for t in ts],
               "per_epoch_s": [round(t / args.epochs, 4) for t in ts],
               "per_step_ms": [round(1e3 * t / (args.epochs * steps), 4) for t in ts],
               "steps_per_epoch": steps, "held_out_accuracy": acc[name]}
        for name, ts, steps in (("fit", times["fit"], steps_fit), ("eager", times["eager"], steps_eager))}
    res["adam_kernel_ms"] = adam_kernel_ms(torch, args.adam_launches)
    if args.al:
        with tempfile.TemporaryDirectory() as out:
            res["active_learning"] = run_al(torch, out)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
