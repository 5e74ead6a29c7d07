"""tip_mc_head against its NumPy restatement (oracle/mc_head_oracle.py): pre-activations bit for bit at the
kernel's edges, probabilities within a stated bound of the float64 softmax, independence from the row and sample
split; and get_pred_and_uncertainty(sampler="head") on the MNIST and IMDB case-study networks."""
import numpy as np
import pytest
import torch

from oracle import mc_head_oracle as MO
from oracle import quantifier_oracle as QO
from simple_tip_b200 import engine as E
from simple_tip_b200.case_studies import imdb, mnist
from simple_tip_b200.core import activations as A
from simple_tip_b200.core import imdb as imdb_inputs

pytestmark = pytest.mark.gpu

ACT = {"l": None, "r": "relu", "s": "softmax"}


def _head(spec, seed=0):
    """spec: (in, [(out, p, act)...]) -> (NumPy layers, device layers)"""
    rng = np.random.default_rng(seed)
    width, host = spec[0], []
    for out, p, act in spec[1]:
        k = (rng.normal(size=(width, out)) / np.sqrt(width)).astype(np.float32)
        b = rng.normal(scale=0.1, size=out).astype(np.float32)
        host.append((k, b, p, ACT[act]))
        width = out
    dev = [(torch.from_numpy(k).cuda(), torch.from_numpy(b).cuda(), p, act) for k, b, p, act in host]
    return host, dev


# (rows, samples, in, layers, row0, sample0): the case studies' heads, every template width, D at 1 and at 8192,
# widths at 64, p = 0 and p = 1, rows and samples that are no multiple of any tile, one sample over many rows
CASES = {
    "mnist": (67, 37, (1600, [(10, 0.5, "s")]), 1000, 5),
    "imdb": (53, 41, (32, [(20, 0.1, "r"), (2, 0.1, "s")]), 0, 0),
    "d1": (300, 7, (1, [(3, 0.5, "s")]), 3, 0),
    "d8192": (5, 9, (8192, [(4, 0.5, "l")]), 0, 190),
    "w64_chain": (19, 13, (40, [(64, 0.3, "r"), (64, 0.2, "r"), (64, 0.0, "l"), (64, 1.0, "s")]), 7, 2),
    "w64_chain_p": (21, 11, (64, [(64, 0.5, "r"), (64, 0.5, "r"), (64, 0.5, "r"), (64, 0.5, "s")]), 0, 0),
    "w64": (33, 70, (100, [(64, 0.5, "r")]), 0, 0),
    "w33": (29, 31, (77, [(33, 0.25, "s")]), 0, 0),
    "w17": (31, 29, (65, [(17, 0.5, "l")]), 0, 0),
    "w13": (17, 101, (63, [(13, 0.5, "s")]), 0, 0),
    "w5": (45, 23, (31, [(5, 0.7, "r")]), 0, 0),
    "w3": (70, 19, (33, [(3, 0.5, "s")]), 0, 0),
    "p0": (23, 17, (50, [(7, 0.0, "s")]), 0, 0),
    "p1": (23, 17, (50, [(7, 1.0, "s")]), 0, 0),
    "s1": (2000, 1, (20, [(5, 0.5, "s")]), 0, 0),
    "tail9": (37, 5, (9, [(9, 0.5, "r"), (1, 0.5, "l")]), 0, 0),
    "tail_odd": (41, 6, (7, [(31, 0.5, "r"), (15, 0.3, "r"), (3, 0.2, "s")]), 0, 0),
}


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _run(name, strided=False):
    rows, samples, spec, row0, sample0 = CASES[name]
    host, dev = _head(spec, seed=len(name))
    h = np.random.default_rng(rows).normal(size=(rows, spec[0])).astype(np.float32)
    hd = torch.from_numpy(h).cuda()
    if strided:        # a view with a row stride above the width
        wide = torch.zeros((rows, spec[0] + 5), device="cuda")
        wide[:, 3:3 + spec[0]] = hd
        hd = wide[:, 3:3 + spec[0]]
    seed = 0xC0FFEE + len(name)
    z = E.mc_head(hd, dev, seed, samples, row0=row0, sample0=sample0, preact=True).cpu().numpy()
    y = E.mc_head(hd, dev, seed, samples, row0=row0, sample0=sample0).cpu().numpy()
    return h, host, dev, seed, z, y, MO.preact(h, host, seed, samples, row0=row0, sample0=sample0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_preactivations_equal_the_restatement_bit_for_bit(name):
    _, host, _, _, z, y, want = _run(name, strided=name in ("mnist", "w13"))
    assert z.shape == want.shape
    assert np.array_equal(_bits(z), _bits(want)), f"{np.sum(_bits(z) != _bits(want))} values differ"
    act = host[-1][3]
    if act == "softmax":
        # relative error of y_c: z_c - m rounded once (|z_c - m| 2^-24 after exp), expf (<= 2 ulp = 4 * 2^-24),
        # C - 1 additions and one division (2^-24 each)
        ref = MO.softmax64(want)
        c = want.shape[2]
        spread = want.max(axis=2, keepdims=True).astype(np.float64) - want
        assert np.all(np.abs(y - ref) <= (c + 4 + spread) * 2.0 ** -24 * ref + 2.0 ** -126)
        assert np.allclose(y.sum(axis=2), 1.0, rtol=0, atol=(c + 4) * 2.0 ** -23)
    elif act == "relu":
        assert np.array_equal(_bits(y), _bits(MO.relu(want)))
    else:
        assert np.array_equal(_bits(y), _bits(want))


def test_p1_drops_everything_and_p0_is_the_plain_layer():
    h, host, _, _, z, _, _ = _run("p1")
    assert np.array_equal(z, np.broadcast_to(host[0][1], z.shape))
    h, host, _, _, z, _, _ = _run("p0")
    assert np.array_equal(z[:, :1], z[:, -1:]) and np.array_equal(z, np.broadcast_to(z[:, :1], z.shape))


@pytest.mark.parametrize("name", ["mnist", "imdb", "w64_chain_p"])
def test_split_rows_and_samples_give_the_same_bits(name):
    rows, samples, spec, row0, sample0 = CASES[name]
    _, dev = _head(spec)
    h = torch.randn(rows, spec[0], device="cuda")
    whole = E.mc_head(h, dev, 9, samples, row0=row0, sample0=sample0)
    parts = torch.cat([torch.cat([E.mc_head(h[r:r + 10], dev, 9, min(7, samples - s), row0=row0 + r,
                                            sample0=sample0 + s) for s in range(0, samples, 7)], dim=1)
                       for r in range(0, rows, 10)], dim=0)
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))
    assert torch.equal(whole, E.mc_head(h, dev, 9, samples, row0=row0, sample0=sample0))
    assert not torch.equal(whole, E.mc_head(h, dev, 10, samples, row0=row0, sample0=sample0))


def test_bad_arguments_are_refused_before_any_launch():
    _, dev = _head((16, [(4, 0.5, "s")]))
    h = torch.randn(8, 16, device="cuda")
    with pytest.raises(ValueError):
        E.mc_head(h.double(), dev, 0, 3)
    with pytest.raises(ValueError):
        E.mc_head(h[:, :15], dev, 0, 3)
    with pytest.raises(ValueError):
        E.mc_head(h, dev, 0, 0)
    with pytest.raises(ValueError):
        E.mc_head(h, [(dev[0][0], dev[0][1], 1.5, "softmax")], 0, 3)
    with pytest.raises(ValueError):
        E.mc_head(h.t(), dev, 0, 3)
    with pytest.raises(ValueError):
        E.mc_head(torch.randn(8, 8193, device="cuda"), dev, 0, 3)


def _mnist_model(n, shift=True):
    torch.manual_seed(0)
    model = mnist.network().cuda()
    x = torch.rand(n, 28, 28, 1, device="cuda")
    if shift:      # balance the classes: the last bias moved by minus the mean logit, so votes are split
        with torch.no_grad():
            logits = model.logits(x)
            model[-1].bias -= logits.mean(dim=0)
    return model, x


def _trunk(model, x, child, batch=128):
    """the head's input as the point pass computes it (same batches, so the same bits)"""
    return A.TransparentModel(model, [child], include_last_layer=False).collect(x, batch)[0].float()


def test_head_vr_is_the_variation_ratio_of_its_own_probabilities(monkeypatch):
    model, x = _mnist_model(700)
    model.train()
    modes = [m.training for m in model.modules()]
    cpu_rng, gpu_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    pred, unc, times = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=60, seed=3, sampler="head")
    assert [m.training for m in model.modules()] == modes
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), gpu_rng)
    assert len(times["VR"]) == 4 and times["VR"][1] > 0
    _, layers = A.mc_head_layers(model)
    probs = E.mc_head(_trunk(model, x, 4), A._head_tensors(layers, x.device), 3, 60).cpu().numpy()
    assert np.array_equal(unc["VR"], QO.variation_ratio(probs)[1])
    # the point results are the default sampler's
    pred_t, unc_t, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=2, seed=3, sampler="torch")
    assert np.array_equal(pred, pred_t)
    for k in ("softmax", "pcs", "softmax_entropy", "deep_gini"):
        assert np.array_equal(unc[k], unc_t[k]), k
    # chunk sizes and repeated calls
    monkeypatch.setattr(A, "MC_ROWS_PER_PASS", 97)
    _, again, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=60, seed=3, sampler="head")
    assert np.array_equal(again["VR"].view(np.uint64), unc["VR"].view(np.uint64))
    monkeypatch.setenv("B200TIP_MC", "head")
    _, env, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=60, seed=3)
    assert np.array_equal(env["VR"], unc["VR"])


def test_p0_head_votes_are_the_point_predictions():
    model, x = _mnist_model(1000)
    model[5].p = 0.0
    pred, unc, _ = A.get_pred_and_uncertainty(model, x, sample_size=20, sampler="head")
    assert np.all(unc["VR"] == 0)
    _, layers = A.mc_head_layers(model)
    probs = E.mc_head(_trunk(model, x, 4, 32), A._head_tensors(layers, x.device), 0, 1).cpu().numpy()
    votes = QO.variation_ratio(probs)[0]
    point = A.TransparentModel(model, [], include_last_layer=True).collect(x, 32)[0].cpu().numpy()
    top2 = np.sort(point, axis=1)[:, -2:]
    near = top2[:, 1] - top2[:, 0] <= 1e-5          # the head sums in its own order: rounding may swap near ties
    assert np.array_equal(votes[~near], pred[~near]) and near.mean() < 0.05


def test_imdb_head_samples_only_the_top_level_dropouts():
    torch.manual_seed(1)
    model = imdb.network().cuda()
    x = torch.from_numpy(np.random.default_rng(2).integers(0, imdb_inputs.VOCAB_SIZE,
                                                           size=(300, imdb_inputs.INPUT_MAXLEN))).float().cuda()
    block = model[2]
    seen = []
    hooks = [m.register_forward_hook(lambda m, i, o: seen.append(m.training)) for m in (block.dropout1, block.dropout2)]
    try:
        _, unc, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=40, seed=5, sampler="head")
    finally:
        for hk in hooks:
            hk.remove()
    assert seen and not any(seen)
    h = _trunk(model, x, 3).cpu().numpy()
    host = [(l.module.kernel.detach().cpu().numpy(), l.module.bias.detach().cpu().numpy(), l.p, l.activation)
            for l in A.mc_head_layers(model)[1]]
    z = MO.preact(h, host, 5, 40)
    gap = np.abs(z[..., 0] - z[..., 1]).min(axis=1)
    clear = gap > 1e-6 * np.abs(z).max(axis=(1, 2))          # no sample within rounding of a tie
    assert clear.mean() > 0.95
    want = QO.variation_ratio(MO.softmax64(z))[1]
    assert np.array_equal(unc["VR"][clear], want[clear])


def test_head_and_torch_samplers_agree_on_mean_vr():
    model, x = _mnist_model(2000)
    _, unc_t, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=200, seed=0, sampler="torch")
    _, unc_h, _ = A.get_pred_and_uncertainty(model, x, batch_size=128, sample_size=200, seed=0, sampler="head")
    assert unc_t["VR"].mean() >= 0.1
    assert abs(unc_t["VR"].mean() - unc_h["VR"].mean()) <= 0.01


def test_default_sampler_is_unchanged(monkeypatch):
    """sampler=None is "torch", and the torch path is the MC loop it always was: replicated batches under torch's
    RNG seeded with `seed`, every dropout module in training mode."""
    monkeypatch.delenv("B200TIP_MC", raising=False)
    model, x = _mnist_model(64)
    _, unc, _ = A.get_pred_and_uncertainty(model, x, batch_size=16, sample_size=30, seed=4)
    _, unc_t, _ = A.get_pred_and_uncertainty(model, x, batch_size=16, sample_size=30, seed=4, sampler="torch")
    assert np.array_equal(unc["VR"], unc_t["VR"])
    model.eval()
    model[5].train()
    samples = []
    with torch.random.fork_rng(devices=[x.device]), torch.no_grad():
        torch.manual_seed(4)
        torch.cuda.manual_seed(4)
        for s in range(0, 64, 16):
            xb = x[s:s + 16]
            samples.append(model(xb.unsqueeze(1).expand(16, 30, 28, 28, 1).reshape(480, 28, 28, 1)).view(16, 30, 10))
    model.eval()
    assert np.array_equal(unc["VR"], QO.variation_ratio(torch.cat(samples).cpu().numpy())[1])
