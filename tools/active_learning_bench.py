"""Where an active-learning run (core/active_learning.evaluate) spends its time; not part of bench.py's line.

    python tools/active_learning_bench.py [--epochs E] [--backends device|default] [--n-train N] [--n-test N]
                                          [--num-selected K]

One `evaluate` call at the MNIST case study's settings (observed_share 0.5, num_selected 1000, 10 classes) on a
PyTorch copy of its CNN (tools/quantifier_bench.mnist_cnn, random weights, last bias shifted to balanced predictions
as in tools/surprise_arm_bench.py), NC layers children [1, 2, 4, 5] and SA layer children [5] as in
tools/coverage_arm_bench.py and tools/surprise_arm_bench.py, 60 k synthetic training inputs, 10 k nominal and 10 k
out-of-distribution ones, labelled with the model's own predictions; every input stays in HBM.  `training_process`
trains a fresh `mnist_cnn` for E epochs (default 1): Adam, batch 128, NLL of the log of the softmax output.

Prints one JSON line with the card's name and power limit, read in the same call, and the wall time of each phase,
each ending in a device synchronise: the split, the original model's evaluation, the fault-predictor, coverage and
surprise selections, the retraining (per model and in total), the retrained models' evaluation and the result files;
and the peak of the torch allocator over the call (`max_memory_allocated` / `max_memory_reserved`).  The fits run
with `B200TIP_{KDE,COV,GMM,KMEANS}=device` unless `--backends default` (sklearn's pc-mlsa fit on 1600-wide rows
takes far longer than the rest).  A warm-up call on slices of the inputs, with one optimizer step per retraining,
comes first.  The result files go to a temporary directory, removed afterwards; nothing is written to the tree.
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
from tools.quantifier_bench import card, mnist_cnn                     # noqa: E402
from tools.surprise_arm_bench import DEVICE_BACKENDS, balanced_model_and_inputs   # noqa: E402

SA_LAYERS = [5]
PHASES = {"_shuffle_and_split_datasets": "split", "_get_fp_selection": "fp_selection",
          "_get_nc_selection": "coverage_selection", "_get_sa_selection": "surprise_selection",
          "_evaluate": "evaluation"}


def make_training_process(torch, epochs, batch_size=128, max_steps=None):
    def train(x, y):
        model = mnist_cnn(torch)
        opt = torch.optim.Adam(model.parameters())
        target = y.argmax(dim=1)
        model.train()
        steps = 0
        for _ in range(epochs):
            perm = torch.randperm(x.shape[0], device=x.device)
            for start in range(0, x.shape[0], batch_size):
                if max_steps is not None and steps == max_steps:
                    break
                idx = perm[start:start + batch_size]
                out = model(x[idx])
                loss = torch.nn.functional.nll_loss(torch.log(out.clamp_min(1e-7)), target[idx])
                opt.zero_grad(set_to_none=True)
                loss.backward()
                opt.step()
                steps += 1
        return model.eval()
    return train


def labelled(torch, model, x):
    with torch.no_grad():
        return torch.cat([model(x[i:i + 8192]).argmax(dim=1) for i in range(0, x.shape[0], 8192)])


def run(torch, AL, model, data, training_process, num_selected, out):
    """evaluate() with every phase's helper and the training process wrapped in a synchronised wall clock."""
    times = {name: [] for name in PHASES.values()}
    times["retraining"] = []
    saved = {name: getattr(AL, name) for name in PHASES}

    def timed(name, fn):
        def call(*args, **kwargs):
            t0 = time.perf_counter()
            res = fn(*args, **kwargs)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            return res
        return call
    for fn_name, phase in PHASES.items():
        setattr(AL, fn_name, timed(phase, saved[fn_name]))
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = AL.evaluate(0, "mnist", model, nc_activation_layers=NC_LAYERS, sa_activation_layers=SA_LAYERS,
                          training_process=timed("retraining", training_process), observed_share=0.5,
                          num_selected=num_selected, num_classes=10, output_folder=out, **data)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        for fn_name, fn in saved.items():
            setattr(AL, fn_name, fn)
    return res, times, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=1)
    ap.add_argument("--backends", choices=["device", "default"], default="device")
    ap.add_argument("--n-train", type=int, default=60_000)
    ap.add_argument("--n-test", type=int, default=10_000)
    ap.add_argument("--num-selected", type=int, default=1000)
    args = ap.parse_args()

    import torch

    from simple_tip_b200.core import active_learning as AL

    if args.backends == "device":
        os.environ.update(DEVICE_BACKENDS)
    else:
        for k in DEVICE_BACKENDS:
            os.environ.pop(k, None)
    res = {"card": card(), "settings": {"epochs": args.epochs, "backends": args.backends, "n_train": args.n_train,
                                        "n_test": args.n_test, "observed_share": 0.5,
                                        "num_selected": args.num_selected, "nc_layers": NC_LAYERS,
                                        "sa_layers": SA_LAYERS}}
    model, train, sets, hist = balanced_model_and_inputs(torch, args.n_train, args.n_test)
    data = {"train_x": train, "train_y": labelled(torch, model, train),
            "nominal_test_x": sets["nominal"], "nominal_test_labels": labelled(torch, model, sets["nominal"]),
            "ood_test_x": sets["ood"], "ood_test_labels": labelled(torch, model, sets["ood"])}
    res["class_histogram"] = hist

    with tempfile.TemporaryDirectory() as out:
        # warm-up on slices (12 k training rows keep pc-lsa's per-class KDE covariance regular): cuDNN plans, the
        # library's modules, first-call allocations, the optimizer's first steps
        warm = {k: v[:12_000] if k.startswith("train") else v[:2000] for k, v in data.items()}
        np.random.seed(0)
        run(torch, AL, model, warm, make_training_process(torch, 1, max_steps=2), 100, out)

        np.random.seed(0)
        torch.cuda.reset_peak_memory_stats()
        (orig, selections, accs), times, wall = run(torch, AL, model, data,
                                                    make_training_process(torch, args.epochs),
                                                    args.num_selected, out)
        files = len(os.listdir(os.path.join(out, "active_learning")))
    retrain, evals = np.array(times["retraining"]), np.array(times["evaluation"][1:])
    phase_sum = sum(sum(v) for v in times.values())
    res["phases_s"] = {
        "split": round(times["split"][0], 4),
        "original_evaluation": round(times["evaluation"][0], 4),
        "fp_selection": round(times["fp_selection"][0], 3),
        "coverage_selection": round(times["coverage_selection"][0], 3),
        "surprise_selection": round(times["surprise_selection"][0], 3),
        "retraining_total": round(float(retrain.sum()), 2),
        "evaluation_total": round(float(evals.sum()), 3),
        "rest": round(wall - phase_sum, 3),
        "wall": round(wall, 2),
    }
    res["retraining_per_model_s"] = {"models": int(retrain.size), "min": round(float(retrain.min()), 3),
                                     "median": round(float(np.median(retrain)), 3),
                                     "max": round(float(retrain.max()), 3),
                                     "steps": args.epochs * -(-(args.n_train + args.num_selected) // 128)}
    res["evaluation_per_model_s"] = {"median": round(float(np.median(evals)), 4)}
    res["peak_gb"] = {"allocated": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                      "reserved": round(torch.cuda.max_memory_reserved() / 1e9, 2)}
    res["result_files"] = files
    res["accuracy"] = {"original": {f"{a}/{b}": v for (a, b), v in orig.items()},
                       "retrained_mean": {f"{a}/{b}": round(float(np.mean([v[a, b] for v in accs.values()])), 4)
                                          for a, b in orig}}
    res["selections"] = len(selections)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
