"""Scoring the fault predictors of a model stack on the GPU: tip_mc_head_stack against M tip_mc_head launches and the
NumPy restatement bit for bit, get_pred_and_uncertainty_stack against the per-model kernels on the stack's own
outputs, the stacked prioritization run against the sequential one, and the stacked accuracies of retrained models."""
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import mc_head_oracle as MO
from simple_tip_b200 import engine as E
from simple_tip_b200.case_studies import imdb, mnist
from simple_tip_b200.case_studies.stacked import stack
from simple_tip_b200.core import active_learning as AL
from simple_tip_b200.core import activations as A
from simple_tip_b200.core import quantifiers as Q
from simple_tip_b200.core.deepgini import DeepGini

pytestmark = pytest.mark.gpu

ACT = {"l": None, "r": "relu", "s": "softmax"}

# (rows, samples, in, layers, row0, sample0): the MNIST and IMDB heads, 3 and 4 layers, rows and samples that are no
# multiple of a block's pairs, nonzero row0 / sample0
HEADS = {
    "mnist": (67, 37, (1600, [(10, 0.5, "s")]), 1000, 5),
    "imdb": (53, 41, (32, [(20, 0.1, "r"), (2, 0.1, "s")]), 3, 0),
    "three": (29, 13, (40, [(33, 0.3, "r"), (17, 0.2, "l"), (5, 0.5, "s")]), 0, 190),
    "four": (21, 11, (64, [(64, 0.5, "r"), (64, 0.5, "r"), (64, 0.0, "l"), (64, 1.0, "s")]), 7, 2),
    "wide1": (45, 23, (31, [(5, 0.7, "r")]), 0, 0),
}


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _stacked_head(models, spec, seed):
    """M heads of one shape: (per-model NumPy layers, stacked device layers)."""
    rng = np.random.default_rng(seed)
    host = [[] for _ in range(models)]
    stacked = []
    width = spec[0]
    for out, p, act in spec[1]:
        k = (rng.normal(size=(models, width, out)) / np.sqrt(width)).astype(np.float32)
        b = rng.normal(scale=0.1, size=(models, out)).astype(np.float32)
        for m in range(models):
            host[m].append((k[m], b[m], p, ACT[act]))
        stacked.append((torch.from_numpy(k).cuda(), torch.from_numpy(b).cuda(), p, ACT[act]))
        width = out
    return host, stacked


def _per_model(layers, m):
    return [(k[m].contiguous(), b[m].contiguous(), p, act) for k, b, p, act in layers]


@pytest.mark.parametrize("preact", [False, True])
@pytest.mark.parametrize("models", [1, 3, 8])
@pytest.mark.parametrize("name", sorted(HEADS))
def test_stack_equals_one_launch_per_model_bit_for_bit(name, models, preact):
    rows, samples, spec, row0, sample0 = HEADS[name]
    _, layers = _stacked_head(models, spec, len(name) + models)
    rng = np.random.default_rng(rows + models)
    # a row window of a wider [M, N, D] tensor: the model stride is not rows * D
    full = torch.from_numpy(rng.normal(size=(models, rows + 9, spec[0])).astype(np.float32)).cuda()
    h = full[:, 4:4 + rows]
    seeds = [0xC0FFEE + 7919 * m for m in range(models)]
    got = E.mc_head_stack(h, layers, seeds, samples, row0=row0, sample0=sample0, preact=preact)
    assert got.shape == (models, rows, samples, spec[1][-1][0])
    for m in range(models):
        want = E.mc_head(h[m], _per_model(layers, m), seeds[m], samples, row0=row0, sample0=sample0, preact=preact)
        assert torch.equal(got[m], want), (m, int((got[m] != want).sum()))


@pytest.mark.parametrize("name", ["mnist", "imdb", "four"])
def test_slice_m_equals_the_restatement_with_model_ms_seed(name):
    rows, samples, spec, row0, sample0 = HEADS[name]
    host, layers = _stacked_head(3, spec, 5)
    h = np.random.default_rng(1).normal(size=(3, rows, spec[0])).astype(np.float32)
    seeds = [3, 2**63 + 5, 0]
    z = E.mc_head_stack(torch.from_numpy(h).cuda(), layers, seeds, samples, row0=row0, sample0=sample0,
                        preact=True).cpu().numpy()
    for m in range(3):
        want = MO.preact(h[m], host[m], seeds[m], samples, row0=row0, sample0=sample0)
        assert np.array_equal(_bits(z[m]), _bits(want)), (m, int(np.sum(_bits(z[m]) != _bits(want))))


def test_more_models_than_one_launch_takes():
    """300 models: two launches of the stacked kernel, each with its own share of the seeds."""
    models, rows, samples = 300, 5, 3
    _, layers = _stacked_head(models, (12, [(4, 0.5, "s")]), 9)
    h = torch.randn(models, rows, 12, device="cuda")
    seeds = list(range(100, 100 + models))
    got = E.mc_head_stack(h, layers, seeds, samples)
    for m in (0, 255, 256, 299):
        assert torch.equal(got[m], E.mc_head(h[m], _per_model(layers, m), seeds[m], samples)), m


def test_a_shared_input_broadcast_over_the_models():
    """h expanded over the model axis (model stride 0) reads every model's rows from the same memory."""
    rows, samples = 70, 9
    _, layers = _stacked_head(4, (1600, [(10, 0.5, "s")]), 2)
    h = torch.randn(rows, 1600, device="cuda")
    got = E.mc_head_stack(h.expand(4, rows, 1600), layers, [1, 1, 2, 3], samples)
    for m in range(4):
        assert torch.equal(got[m], E.mc_head(h, _per_model(layers, m), [1, 1, 2, 3][m], samples))
    assert not torch.equal(got[1], got[2])


def test_wrapper_refuses_bad_arguments():
    _, layers = _stacked_head(2, (16, [(4, 0.5, "s")]), 0)
    h = torch.randn(2, 5, 16, device="cuda")
    with pytest.raises(ValueError, match="seeds"):
        E.mc_head_stack(h, layers, [0], 3)
    with pytest.raises(ValueError, match="3-D"):
        E.mc_head_stack(h[0], layers, [0, 1], 3)
    with pytest.raises(ValueError, match="models"):
        E.mc_head_stack(torch.randn(3, 5, 16, device="cuda"), layers, [0, 1, 2], 3)
    with pytest.raises(ValueError, match="column stride"):
        E.mc_head_stack(h.transpose(1, 2), layers, [0, 1], 3)
    with pytest.raises(ValueError, match="samples"):
        E.mc_head_stack(h, layers, [0, 1], 0)


# ---- get_pred_and_uncertainty_stack --------------------------------------------------------------------------------------
def _networks(module, count, seed):
    torch.manual_seed(seed)
    return [module.network().cuda().eval() for _ in range(count)]


def _inputs(name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "mnist":
        return torch.from_numpy(rng.random((n, 28, 28, 1), dtype=np.float32)).cuda()
    return torch.from_numpy(rng.integers(0, 2000, size=(n, 100)).astype(np.int32)).cuda()


def _stack_outputs(net, x, batch_size, at):
    """The stack's probabilities [M, N, C] and its head input [M, N, D], batch by batch as the scoring runs."""
    m = len(net.sources)
    trunk = []
    hook = list(net.children())[at].register_forward_pre_hook(lambda _m, inp: trunk.append(inp[0].detach()))
    try:
        with torch.no_grad():
            probs = torch.cat([net(net.stack_inputs([x[s:s + batch_size]] * m)) for s in range(0, len(x), batch_size)],
                              dim=1)
    finally:
        hook.remove()
    return probs, torch.cat(trunk, dim=1)


@pytest.mark.parametrize("name, module, n", [("mnist", mnist, 300), ("imdb", imdb, 200)])
def test_head_sampler_equals_the_per_model_kernels_on_the_stacks_outputs(name, module, n):
    models = _networks(module, 3, 11)
    net = stack(models).eval()
    x = _inputs(name, n, 4)
    seeds = [0, 17, 2**40]
    got = A.get_pred_and_uncertainty_stack(net, x, sample_size=60, seeds=seeds, sampler="head")
    assert len(got) == 3
    at, head = A.mc_head_layers_stack(net)
    probs, h = _stack_outputs(net, x, 32, at)
    layers = A._head_tensors(head, h.device)
    for m, (pred, unc, times) in enumerate(got):
        assert list(unc) == ["softmax", "pcs", "softmax_entropy", "deep_gini", "VR"]
        assert set(times) == set(unc) and all(len(t) == 4 for t in times.values())
        for q in (Q.MaxSoftmax, Q.PredictionConfidenceScore, Q.SoftmaxEntropy, DeepGini):
            q_pred, values = q.calculate(probs[m])
            np.testing.assert_array_equal(pred, q_pred)
            name = q.aliases()[0].replace("custom::", "")
            np.testing.assert_array_equal(unc[name], q.cast_conf_or_unc(False, values))
        samples = E.mc_head(h[m].contiguous(), _per_model(layers, m), seeds[m], 60)
        _, vr = Q.VariationRatio.calculate(samples)
        np.testing.assert_array_equal(unc["VR"], vr)
    # against each unstacked model on its own: the same draws on its own forward's head input
    for m, model in enumerate(net.unstack()):
        _, unc, _ = A.get_pred_and_uncertainty(model, x, sample_size=60, seed=seeds[m], sampler="head")
        assert abs(unc["VR"].mean() - got[m][1]["VR"].mean()) <= 0.01


def test_torch_sampler_on_a_stack_and_the_modes_it_restores():
    models = _networks(mnist, 2, 3)
    net = stack(models).train()
    x = _inputs("mnist", 40, 1)
    got = A.get_pred_and_uncertainty_stack(net, x, sample_size=20, sampler="torch")
    assert all(m.training for m in net.modules())
    probs, _ = _stack_outputs(net.eval(), x, 32, A.mc_head_layers_stack(net)[0])
    for m, (pred, unc, times) in enumerate(got):
        np.testing.assert_array_equal(pred, probs[m].argmax(dim=1).cpu().numpy())
        assert unc["VR"].shape == (40,) and 0 <= unc["VR"].min() and unc["VR"].max() < 1
        assert len(times["VR"]) == 4
    again = A.get_pred_and_uncertainty_stack(net, x, sample_size=20, sampler="torch")
    for (_, a, _), (_, b, _) in zip(got, again):
        np.testing.assert_array_equal(a["VR"], b["VR"])


# ---- the prioritization run ------------------------------------------------------------------------------------------------
def _blocks(rng, n):
    """MNIST-shaped uint8 images whose class is the 7 x 7 block (of a 4 x 4 grid) that is bright."""
    labels = rng.integers(0, 10, size=n)
    x = rng.integers(0, 90, size=(n, 28, 28), dtype=np.uint8)
    for i, c in enumerate(labels):
        r, k = divmod(int(c), 4)
        x[i, 7 * r:7 * r + 7, 7 * k:7 * k + 7] += np.uint8(160)
    return x, labels.astype(np.uint8)


APFD_TOLERANCE = 0.02       # the fault predictors' APFDs: stacked against per-model forwards, head sampler


@pytest.fixture(scope="module")
def prio_runs(tmp_path_factory):
    mp = pytest.MonkeyPatch()
    for k, v in {"B200TIP_KDE": "device", "B200TIP_COV": "device", "B200TIP_GMM": "device",
                 "B200TIP_KMEANS": "device", "B200TIP_MC": "head"}.items():
        mp.setenv(k, v)
    try:
        rng = np.random.default_rng(2)
        nominal = (_blocks(rng, 1200), _blocks(rng, 200))
        data = tmp_path_factory.mktemp("datasets")
        cx, cl = _blocks(rng, 200)
        np.save(data / "mnist_c_images.npy", np.expand_dims(255 - cx, -1))
        np.save(data / "mnist_c_labels.npy", cl.astype(np.int64))
        datasets = mnist.load_datasets(nominal, str(data))
        out = str(tmp_path_factory.mktemp("assets"))
        cs = mnist.MnistCaseStudy(out, datasets, epochs=1)
        np.random.seed(0)
        cs.train([0, 1, 2], stacked=True)
        res = {}
        for stacked in (False, True):
            cs.output_folder = str(tmp_path_factory.mktemp(f"prio_{stacked}"))
            os.makedirs(os.path.dirname(cs.model_path(0)))
            for i in (0, 1, 2):
                shutil.copyfile(os.path.join(out, "models", "mnist", f"model_{i}.pt"), cs.model_path(i))
            np.random.seed(5)
            res[stacked] = (cs.run_prio_eval([0, 1, 2], stacked=stacked, stack_size=2 if stacked else None),
                            cs.output_folder)
    finally:
        mp.undo()
    return res


def test_stacked_prioritization_writes_the_sequential_files(prio_runs):
    (seq, seq_dir), (stk, stk_dir) = prio_runs[False], prio_runs[True]
    for sub in ("priorities", "times"):
        assert sorted(os.listdir(os.path.join(seq_dir, sub))) == sorted(os.listdir(os.path.join(stk_dir, sub)))
    files = sorted(os.listdir(os.path.join(seq_dir, "priorities")))
    assert any("uncertainty_VR" in f for f in files)
    fault_predictors = ("is_misclassified", "uncertainty_")
    for f in files:
        if any(k in f for k in fault_predictors):
            continue
        a, b = (np.load(os.path.join(d, "priorities", f)) for d in (seq_dir, stk_dir))
        np.testing.assert_array_equal(a, b, err_msg=f)
    assert list(seq) == list(stk) == [0, 1, 2]
    for model_id in seq:
        for ds in ("nominal", "ood"):
            assert list(seq[model_id][ds]) == list(stk[model_id][ds])
            for approach, apfd in seq[model_id][ds].items():
                if approach in ("softmax", "pcs", "softmax_entropy", "deep_gini", "VR"):
                    assert abs(apfd - stk[model_id][ds][approach]) <= APFD_TOLERANCE, (model_id, ds, approach)
                else:
                    assert apfd == stk[model_id][ds][approach], (model_id, ds, approach)


# ---- active learning's retrained models ------------------------------------------------------------------------------------
def test_stacked_accuracies_equal_accuracy_on_the_stacked_probabilities():
    models = _networks(mnist, 80, 21)
    net = stack(models).eval()
    x = _inputs("mnist", 333, 2)
    y = torch.from_numpy(np.random.default_rng(3).integers(0, 10, 333)).cuda()
    got = AL.accuracies_stack(net, x, y, batch_size=128)
    with torch.no_grad():
        probs = torch.cat([net(net.stack_inputs([x[s:s + 128]] * 80)) for s in range(0, 333, 128)], dim=1)

    class Fixed(torch.nn.Module):
        """One model's slice of the stacked probabilities, served in order."""

        def __init__(self, p):
            super().__init__()
            self.p, self.at, self.w = p, 0, torch.nn.Parameter(torch.zeros(1, device=p.device))

        def forward(self, xb):
            out = self.p[self.at:self.at + xb.shape[0]]
            self.at += xb.shape[0]
            return out

    for m in range(80):
        assert got[m] == AL.accuracy(Fixed(probs[m]), x, y, batch_size=128), m
    datasets = {("nominal", "observed"): (x[:100], y[:100]), ("ood", "future"): (x[100:], y[100:])}
    per_model = AL._evaluate_stack(models, datasets, 10, batch_size=128)
    assert len(per_model) == 80 and all(list(r) == list(datasets) for r in per_model)
    for m in (0, 79):
        for key, (xs, ys) in datasets.items():
            assert per_model[m][key] == AL.accuracies_stack(net, xs, ys, 128)[m]
