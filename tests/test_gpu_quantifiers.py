"""GPU parity of the uncertainty quantifiers (core/quantifiers.py, core/activations.get_pred_and_uncertainty) against
oracle/quantifier_oracle.py.

Tolerances: predictions, max softmax, PCS and the variation ratio are bit-exact.  Softmax entropy sums in NumPy's
pairwise order on both sides and only log2 differs (at most an ulp on each side), so a row stays within
4 * (2 + ceil(log2 C)) * u * sum |q log2 q|, u the unit roundoff of the input dtype."""
import math

import numpy as np
import pytest

from oracle import np_oracle
from oracle import quantifier_oracle as QO

pytestmark = pytest.mark.gpu


def _torch():
    import torch

    return torch


def _softmax_rows(n, c, dt, seed):
    """Dirichlet rows plus the awkward cases: saturated one-hot rows, a repeated maximum, exact zeros."""
    rng = np.random.default_rng(seed)
    p = rng.dirichlet(np.full(c, 0.5), size=n)
    if n >= 8:
        p[0] = 0
        p[0, c - 1] = 1                                   # one-hot, last class
        p[1] = 0
        p[1, 0] = 1                                       # one-hot, first class
        p[2] = 1.0 / c                                    # every class tied
        p[3, :] = p[3] / 2
        p[3, 0] = p[3, c - 1] = 0.25                      # repeated maximum
        p[4, : c // 2] = 0                                # exact zeros
    return np.ascontiguousarray(p.astype(dt))


def _entropy_bound(p):
    q = np.where(p == 0, p.dtype.type(1e-20), p).astype(np.float64)
    u = np.finfo(p.dtype).eps / 2
    return 4 * (2 + math.ceil(math.log2(p.shape[1]))) * u * np.sum(np.abs(q * np.log2(q)), axis=1)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("c", [2, 10, 100, 1000, 5000])
def test_point_quantifiers_against_the_oracle(dt, c):
    from simple_tip_b200.core.quantifiers import MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy

    p = _softmax_rows(1000 + 37 if c < 5000 else 300 + 5, c, dt, seed=c)
    wp = np.argmax(p, axis=1)
    for cls, oracle in ((MaxSoftmax, QO.max_softmax), (PredictionConfidenceScore, QO.pcs)):
        pred, val = cls.calculate(p)
        _, want = oracle(p)
        assert pred.dtype == np.int64 and np.array_equal(pred, wp), cls
        assert val.dtype == dt and np.array_equal(val, want), cls
    pred, ent = SoftmaxEntropy.calculate(p)
    _, want = QO.softmax_entropy(p)
    assert np.array_equal(pred, wp) and ent.dtype == dt
    err = np.abs(ent.astype(np.float64) - want.astype(np.float64))
    assert np.all(err <= _entropy_bound(p)), (np.max(err), c)


def test_empty_input_and_one_class():
    from simple_tip_b200.core.quantifiers import (MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy,
                                                  VariationRatio)

    for cls in (MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy):
        pred, val = cls.calculate(np.zeros((0, 10), dtype=np.float32))
        assert pred.shape == (0,) and val.shape == (0,) and val.dtype == np.float32
    pred, vr = VariationRatio.calculate(np.zeros((0, 4, 10)))
    assert pred.shape == (0,) and vr.shape == (0,) and vr.dtype == np.float64
    with pytest.raises(ValueError):
        PredictionConfidenceScore.calculate(np.ones((5, 1), dtype=np.float32))
    pred, val = MaxSoftmax.calculate(np.ones((5, 1), dtype=np.float32))
    assert np.array_equal(pred, np.zeros(5)) and np.array_equal(val, np.ones(5, dtype=np.float32))


def test_cuda_tensors_give_the_numpy_bits():
    torch = _torch()
    from simple_tip_b200.core.quantifiers import (MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy,
                                                  VariationRatio)

    dev = torch.device("cuda", 0)
    for dt in (np.float32, np.float64):
        p = _softmax_rows(777, 10, dt, seed=5)
        for cls in (MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy):
            a, b = cls.calculate(p), cls.calculate(torch.from_numpy(p).to(dev))
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[1].dtype == b[1].dtype
    # half-precision CUDA tensors are widened to float32
    h = torch.from_numpy(_softmax_rows(300, 10, np.float32, seed=6)).to(dev).half()
    for cls in (MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy):
        a, b = cls.calculate(h), cls.calculate(h.float().cpu().numpy())
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[1].dtype == np.float32
    s = np.random.default_rng(7).dirichlet(np.ones(10), size=(50, 20)).astype(np.float32)
    a, b = VariationRatio.calculate(s), VariationRatio.calculate(torch.from_numpy(s).to(dev))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("n,s,c", [(1000 + 37, 200, 10), (300, 4, 3), (129, 7, 2), (64, 33, 100), (20, 5, 5000),
                                   (6, 5, 13000)])        # c > 12288: the votes are counted in global memory
def test_variation_ratio_against_the_oracle(dt, n, s, c):
    from simple_tip_b200.core.quantifiers import VariationRatio

    rng = np.random.default_rng(n + s + c)
    votes = rng.integers(0, min(c, 3), size=(n, s))          # few classes voted: many ties of the mode
    p = rng.dirichlet(np.ones(c), size=(n, s)) * 0.5
    np.put_along_axis(p, votes[..., None], 0.9, axis=2)
    p[0] = 0
    p[0, :, c - 1] = 1                                          # saturated: every sample one-hot
    p = p.astype(dt)
    pred, vr = VariationRatio.calculate(p)
    wp, wv = QO.variation_ratio(p)
    assert pred.dtype == np.int64 and np.array_equal(pred, wp)
    assert vr.dtype == np.float64 and np.array_equal(vr, wv)


def test_votes_reject_what_the_kernel_cannot_read():
    torch = _torch()
    from simple_tip_b200.core.quantifiers import Votes

    dev = torch.device("cuda", 0)
    p = torch.rand(10, 4, 6, device=dev)
    with pytest.raises(ValueError):
        Votes(10, 6, "cpu")                                     # counts off the current CUDA device
    votes = Votes(10, 6, "cuda")
    for bad in (p.cpu(), p.cpu().numpy(), p.to(torch.float16), p.to(torch.int32)):
        with pytest.raises(ValueError):
            votes.add(bad, 4, sample_stride=6, row_stride=24)
    with pytest.raises(ValueError):
        votes.add(p, 5, sample_stride=6, row_stride=24)         # one sample more than the tensor holds
    with pytest.raises(ValueError):
        votes.add(p[5:], 4, sample_stride=6, row_stride=24)     # rows 0..9 of a view that has 5
    with pytest.raises(ValueError):
        votes.add(p, 4, sample_stride=6, row_stride=24, row0=8, rows=3)
    assert int(votes.counts.sum()) == 0                          # nothing was launched
    votes.add(p[5:], 4, sample_stride=6, row_stride=24, row0=5, rows=5)
    assert int(votes.counts[:5].sum()) == 0 and int(votes.counts[5:].sum()) == 20


def test_chunked_votes_equal_one_dense_call():
    torch = _torch()
    from simple_tip_b200.core.quantifiers import Votes

    dev = torch.device("cuda", 0)
    n, s, c = 333, 50, 10
    p = torch.from_numpy(np.random.default_rng(8).dirichlet(np.ones(c), size=(n, s)).astype(np.float32)).to(dev)
    dense = Votes(n, c, dev)
    dense.add(p, s, sample_stride=c, row_stride=s * c)
    chunked = Votes(n, c, dev)
    for r0, r1 in ((0, 100), (100, 333)):                       # rows in two chunks, samples in three
        for s0, s1 in ((0, 7), (7, 31), (31, 50)):
            chunked.add(p[r0:, s0:], s1 - s0, sample_stride=c, row_stride=s * c, row0=r0,
                        rows=r1 - r0)
    assert torch.equal(dense.counts, chunked.counts)
    assert int(dense.counts.sum()) == n * s
    a, b = dense.finish(s), chunked.finish(s)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def _mlp(torch, p_drop, dropout=True, device="cuda"):
    layers = [torch.nn.Linear(8, 32), torch.nn.BatchNorm1d(32), torch.nn.ReLU()]
    if dropout:
        layers.append(torch.nn.Dropout(p_drop))
    layers += [torch.nn.Linear(32, 5), torch.nn.Softmax(dim=1)]
    torch.manual_seed(0)
    model = torch.nn.Sequential(*layers).to(device)
    with torch.no_grad():                                       # non-trivial running statistics
        model[1].running_mean.uniform_(-0.5, 0.5)
        model[1].running_var.uniform_(0.5, 2.0)
    return model


def test_get_pred_and_uncertainty_mc_dropout():
    torch = _torch()
    from simple_tip_b200.core.activations import get_pred_and_uncertainty

    model = _mlp(torch, 0.3)
    model.train()
    model[4].eval()                                             # a mixed state, to be restored as it was
    flags = [m.training for m in model.modules()]
    bn = {k: v.clone() for k, v in model[1].state_dict().items()}
    x = torch.from_numpy(np.random.default_rng(9).normal(size=(100, 8)).astype(np.float32)).to("cuda")
    outputs = []
    hook = model.register_forward_hook(lambda _m, _i, out: outputs.append(out.detach().clone()))
    cpu_rng, gpu_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    try:
        pred, unc, times = get_pred_and_uncertainty(model, x, batch_size=32, sample_size=16, seed=3)
    finally:
        hook.remove()
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), gpu_rng)
    assert [m.training for m in model.modules()] == flags
    assert all(torch.equal(v, bn[k]) for k, v in model[1].state_dict().items())
    assert set(unc) == {"softmax", "pcs", "softmax_entropy", "deep_gini", "VR"} and set(times) == set(unc)
    assert all(len(t) == 4 and t[0] == 0 and t[3] == 0 and t[1] >= 0 and t[2] >= 0 for t in times.values())

    # point pass: 4 batches of the eval-mode model; then one MC pass per batch (32 x 16 rows <= the pass budget)
    probs = torch.cat(outputs[:4]).cpu().numpy()
    want = QO.study_uncertainties(probs)
    assert np.array_equal(pred, np.argmax(probs, axis=1)) and pred.dtype == np.int64
    for k in ("softmax", "pcs", "deep_gini"):
        assert np.array_equal(unc[k], want[k]), k
    assert np.all(np.abs(unc["softmax_entropy"] - want["softmax_entropy"]) <= _entropy_bound(probs))
    assert len(outputs) == 8
    samples = np.concatenate([o.view(-1, 16, 5).cpu().numpy() for o in outputs[4:]])
    assert samples.shape == (100, 16, 5)
    assert not np.array_equal(samples[:, 0], samples[:, 1])     # the replicas drew different dropout masks
    assert np.array_equal(unc["VR"], QO.variation_ratio(samples)[1])

    again = get_pred_and_uncertainty(model, x, batch_size=32, sample_size=16, seed=3)
    assert all(np.array_equal(again[1][k], unc[k]) for k in unc)
    # the default sample size, passes of 32 x 200 rows
    _, unc200, _ = get_pred_and_uncertainty(model, x.cpu().numpy(), seed=3)
    assert unc200["VR"].shape == (100,) and np.all((unc200["VR"] >= 0) & (unc200["VR"] < 0.8))


def test_get_pred_and_uncertainty_without_sampling_noise():
    torch = _torch()
    from simple_tip_b200.core.activations import get_pred_and_uncertainty

    x = torch.from_numpy(np.random.default_rng(10).normal(size=(70, 8)).astype(np.float32)).to("cuda")
    _, unc, _ = get_pred_and_uncertainty(_mlp(torch, 0.0), x, sample_size=10)
    assert np.array_equal(unc["VR"], np.zeros(70))                # p = 0: every sample votes the point prediction
    _, unc, times = get_pred_and_uncertainty(_mlp(torch, 0.0, dropout=False), x, sample_size=10)
    assert "VR" not in unc and "VR" not in times and len(unc) == 4


def test_result_files_give_the_oracle_apfd(tmp_path):
    torch = _torch()
    from simple_tip_b200.core import results as R
    from simple_tip_b200.core.activations import get_pred_and_uncertainty
    from src.core.apfd import apfd_from_order

    model = _mlp(torch, 0.5)
    x = torch.from_numpy(np.random.default_rng(11).normal(size=(400, 8)).astype(np.float32)).to("cuda")
    outputs = []
    hook = model.register_forward_hook(lambda _m, _i, out: outputs.append(out.detach().clone()))
    try:
        pred, unc, _ = get_pred_and_uncertainty(model, x, batch_size=100, sample_size=20, seed=0)
    finally:
        hook.remove()
    probs = torch.cat(outputs[:4]).cpu().numpy()
    samples = np.concatenate([o.view(-1, 20, 5).cpu().numpy() for o in outputs[4:]])
    labels = np.random.default_rng(12).integers(0, 5, size=400)
    mis = pred != labels
    out = str(tmp_path)
    R.persist(out, "toy", "nominal", "is_misclassified", 0, mis)
    for name, values in unc.items():
        R.persist(out, "toy", "nominal", f"uncertainty_{name}", 0, values)
    apfd = R.load_apfd_values(out, "toy", "nominal")
    want = QO.study_uncertainties(probs, samples)
    assert set(apfd) == {"softmax", "pcs", "softmax_entropy", "deep_gini", "VR"}
    for name, values in want.items():
        expect = apfd_from_order(mis, np.argsort(-values))
        if name == "softmax_entropy":
            assert abs(apfd[name][0] - expect) <= 1e-6
        else:
            assert apfd[name][0] == expect, name
    assert np.array_equal(want["deep_gini"], np_oracle.deepgini_oracle(probs)[1])


def test_get_pred_and_uncertainty_with_a_host_model():
    """A model on the host runs there; its outputs are scored on the current CUDA device, MC passes included."""
    torch = _torch()
    from simple_tip_b200.core.activations import get_pred_and_uncertainty

    model = _mlp(torch, 0.3, device="cpu")
    x = np.random.default_rng(13).normal(size=(70, 8)).astype(np.float32)
    outputs = []
    hook = model.register_forward_hook(lambda _m, _i, out: outputs.append(out.detach().clone()))
    cpu_rng = torch.get_rng_state()
    try:
        pred, unc, _ = get_pred_and_uncertainty(model, x, batch_size=32, sample_size=12, seed=1)
    finally:
        hook.remove()
    assert torch.equal(torch.get_rng_state(), cpu_rng)
    assert all(p.device.type == "cpu" for p in model.parameters()) and model.training
    assert len(outputs) == 6 and all(o.device.type == "cpu" for o in outputs)
    probs = torch.cat(outputs[:3]).numpy()
    want = QO.study_uncertainties(probs)
    assert np.array_equal(pred, np.argmax(probs, axis=1))
    for k in ("softmax", "pcs", "deep_gini"):
        assert np.array_equal(unc[k], want[k]), k
    samples = np.concatenate([o.view(-1, 12, 5).numpy() for o in outputs[3:]])
    assert samples.shape == (70, 12, 5)
    assert np.array_equal(unc["VR"], QO.variation_ratio(samples)[1])
    again = get_pred_and_uncertainty(model, x, batch_size=32, sample_size=12, seed=1)
    assert np.array_equal(again[1]["VR"], unc["VR"])


def test_get_pred_and_uncertainty_needs_inputs():
    torch = _torch()
    from simple_tip_b200.core.activations import get_pred_and_uncertainty

    with pytest.raises(ValueError):
        get_pred_and_uncertainty(_mlp(torch, 0.3), np.zeros((0, 8), dtype=np.float32))
