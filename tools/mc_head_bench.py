"""What the MC-dropout variation ratio costs with the head sampler against the torch sampler; not part of bench.py.

    python tools/mc_head_bench.py [--rounds R] [--launches K] [--imdb-torch-n N] [--prio]

`get_pred_and_uncertainty` (S = 200, batch = the case study's prediction badge size, 128) with sampler="torch"
against sampler="head", on:

  * the MNIST case-study CNN (seeded weights, last bias shifted by minus the mean logit so the votes split),
    10 000 seeded U(0, 1) images;
  * the IMDB case-study transformer (seeded weights), 25 000 seeded synthetic reviews of 100 token ids (the first 40
    padding).  200 transformer forwards per review take long with the torch sampler, so it is timed on the first
    --imdb-torch-n reviews (default 2 500), and the head sampler on both that slice and all 25 000.

After a warm-up of both samplers, R rounds alternate the two; every wall time ends in a device synchronise, and the
sampling and vote times are the call's own times["VR"].  Then `tip_mc_head` alone on the MNIST head (10 000 rows of
the trunk, 200 samples, one launch and the sampler's 8 192-row chunk), by CUDA events around K launches: ms per
launch, multiply-adds per second, and the share of the FP32 data-sheet rate (67 TFLOP/s for an H100 SXM at 700 W =
33.5 T FP32 instructions/s; the kernel issues one multiply and one add per multiply-add, so its floor is
2 x multiply-adds / 33.5e12 s).  --prio: one tools/prioritization_bench.py run with B200TIP_MC=head (its own JSON
line is embedded).

Prints one JSON line with the card's name and power limit, read in the same call.  Nothing is written to the tree.
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

from tools.quantifier_bench import card                                   # noqa: E402

FP32_INSTR_PER_S = 33.5e12        # H100 SXM data sheet: 67 TFLOP/s FP32, an FMA counted as two


def synced(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def mnist_case(torch, n):
    from simple_tip_b200.case_studies import mnist

    torch.manual_seed(0)
    model = mnist.network().cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((n, 28, 28, 1), device="cuda", generator=g)
    with torch.no_grad():
        model[-1].bias -= torch.cat([model.logits(x[i:i + 8192]) for i in range(0, n, 8192)]).mean(dim=0)
    return model, x


def imdb_case(torch, n):
    from simple_tip_b200.case_studies import imdb
    from simple_tip_b200.core import imdb as inputs

    torch.manual_seed(0)
    model = imdb.network().cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(1, inputs.VOCAB_SIZE, (n, inputs.INPUT_MAXLEN), device="cuda", generator=g, dtype=torch.int32)
    x[:, :40] = 0
    return model, x


def samplers(torch, A, model, x, rounds, samplers=("torch", "head")):
    """{sampler: {"wall_s": [...], "sampling_s": [...], "vote_s": [...], "mean_vr": ...}} over alternating rounds."""
    res = {s: {"wall_s": [], "sampling_s": [], "vote_s": []} for s in samplers}
    for s in samplers:            # warm-up
        A.get_pred_and_uncertainty(model, x[:256], batch_size=128, sample_size=200, sampler=s)
    for _ in range(rounds):
        for s in samplers:
            (_, unc, times), wall = synced(torch, lambda: A.get_pred_and_uncertainty(
                model, x, batch_size=128, sample_size=200, sampler=s))
            res[s]["wall_s"].append(round(wall, 4))
            res[s]["sampling_s"].append(round(times["VR"][1], 4))
            res[s]["vote_s"].append(round(times["VR"][2], 4))
            res[s]["mean_vr"] = round(float(unc["VR"].mean()), 5)
    return res


def kernel_alone(torch, A, E, model, x, launches):
    first, head = A.mc_head_layers(model)
    trunk = A.TransparentModel(model, [first - 1], include_last_layer=False).collect(x, 128)[0].contiguous()
    layers = A._head_tensors(head, trunk.device)
    out = {}
    for rows in (trunk.shape[0], min(A.MC_ROWS_PER_PASS, trunk.shape[0])):
        h = trunk[:rows]
        buf = torch.empty((rows, 200, layers[-1][0].shape[1]), device="cuda")
        for _ in range(3):
            E.mc_head(h, layers, 0, 200, out=buf)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(launches):
            E.mc_head(h, layers, 0, 200, out=buf)
        end.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(end) / launches
        mads = sum(rows * 200 * k.shape[0] * k.shape[1] for k, _, _, _ in layers)
        floor_ms = 2 * mads / FP32_INSTR_PER_S * 1e3
        out[f"rows_{rows}"] = {"ms": round(ms, 4), "multiply_adds": mads, "mad_per_s": f"{mads / ms * 1e3:.3e}",
                               "floor_ms": round(floor_ms, 4), "share_of_fp32_rate": round(floor_ms / ms, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--mnist-n", type=int, default=10_000)
    ap.add_argument("--imdb-n", type=int, default=25_000)
    ap.add_argument("--imdb-torch-n", type=int, default=2_500)
    ap.add_argument("--prio", action="store_true")
    args = ap.parse_args()

    import torch

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core import activations as A

    if not torch.cuda.is_available():
        raise SystemExit("mc_head_bench needs a CUDA device")
    res = {"card": card(), "samples": 200}
    model, x = mnist_case(torch, args.mnist_n)
    res["mnist"] = {"n": args.mnist_n, **samplers(torch, A, model, x, args.rounds)}
    res["mnist_kernel"] = kernel_alone(torch, A, E, model, x, args.launches)
    model, x = imdb_case(torch, args.imdb_n)
    res["imdb_slice"] = {"n": args.imdb_torch_n, **samplers(torch, A, model, x[:args.imdb_torch_n], args.rounds)}
    res["imdb_full"] = {"n": args.imdb_n, "torch": "not measured (timed on the slice)",
                        **samplers(torch, A, model, x, args.rounds, samplers=("head",))}
    if args.prio:
        env = dict(os.environ, B200TIP_MC="head")
        run = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "prioritization_bench.py")], env=env,
                             capture_output=True, text=True, cwd=ROOT)
        lines = [l for l in run.stdout.splitlines() if l.startswith("{")]
        res["prioritization_B200TIP_MC_head"] = json.loads(lines[-1]) if lines else run.stderr[-2000:]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
