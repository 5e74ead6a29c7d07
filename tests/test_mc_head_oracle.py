"""The MC-dropout head's host side without a GPU: the oracle's counter-based draws (keep rates, distinct streams,
independence from the row / sample split), the head parser on the case studies' networks and plain torch modules,
and tip_mc_head's argument checks through the C ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as KO
from oracle import mc_head_oracle as MO
from simple_tip_b200 import _lib
from simple_tip_b200.case_studies import base, imdb, mnist
from simple_tip_b200.core import activations as A


def test_draws_are_the_documented_splitmix_chain():
    seed, layer, row, sample = 0x1234_5678_9ABC_DEF0, 2, 70_001, 199
    key = KO.km_mix(KO.km_mix(KO.km_mix(KO.km_mix(seed) ^ layer) ^ row) ^ sample)
    u = MO.draws(seed, layer, np.array([row]), np.array([sample]), 7)[0, 0]
    for j in range(7):
        w = KO.km_mix(key ^ (j >> 1))
        assert int(u[j]) == (w >> 32 if j & 1 else w & 0xFFFFFFFF)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate_within_six_sigma(p):
    rows, samples, units = np.arange(50), np.arange(200), 128         # 1.28e6 draws
    drop = MO.dropped(7, 0, rows, samples, units, p)
    n = drop.size
    assert n >= 10 ** 6
    assert abs(drop.sum() - n * p) <= 6 * np.sqrt(n * p * (1 - p))


def test_thresholds_and_scales():
    assert MO.threshold(0.5) == 2 ** 31 and MO.threshold(0.0) == 0 and MO.threshold(1.0) == 2 ** 32
    assert MO.scale(0.5) == np.float32(2.0) and MO.scale(0.0) == np.float32(1.0)
    assert MO.scale(0.1) == np.float32(1.0) / np.float32(0.9)
    assert MO.dropped(3, 0, np.arange(4), np.arange(5), 9, 1.0).all()
    assert not MO.dropped(3, 0, np.arange(4), np.arange(5), 9, 0.0).any()


def test_distinct_keys_give_distinct_streams():
    base_u = MO.draws(11, 0, np.array([5]), np.array([3]), 64)[0, 0]
    for layer, row, sample, seed in ((1, 5, 3, 11), (0, 6, 3, 11), (0, 5, 4, 11), (0, 5, 3, 12), (0, 3, 5, 11)):
        other = MO.draws(seed, layer, np.array([row]), np.array([sample]), 64)[0, 0]
        assert np.mean(base_u == other) < 0.1, (layer, row, sample, seed)
    u = MO.draws(11, 0, np.arange(30), np.arange(30), 16).reshape(900, 16)
    assert len({r.tobytes() for r in u}) == 900


def test_chunked_and_whole_calls_draw_the_same_masks():
    rows, samples = np.arange(100, 137), np.arange(0, 23)
    whole = MO.dropped(5, 1, rows, samples, 33, 0.5)
    parts = np.concatenate([np.concatenate([MO.dropped(5, 1, rows[r:r + 10], samples[s:s + 7], 33, 0.5)
                                            for s in range(0, 23, 7)], axis=1) for r in range(0, 37, 10)], axis=0)
    assert np.array_equal(whole, parts)
    rng = np.random.default_rng(0)
    layers = [(rng.normal(size=(33, 5)).astype(np.float32), rng.normal(size=5).astype(np.float32), 0.5, "relu"),
              (rng.normal(size=(5, 3)).astype(np.float32), rng.normal(size=3).astype(np.float32), 0.25, "softmax")]
    h = rng.normal(size=(37, 33)).astype(np.float32)
    z = MO.preact(h, layers, 5, 23, row0=100)
    split = np.concatenate([MO.preact(h[r:r + 10], layers, 5, 23, row0=100 + r) for r in range(0, 37, 10)])
    tail = MO.preact(h, layers, 5, 9, row0=100, sample0=14)
    assert np.array_equal(z, split) and np.array_equal(z[:, 14:], tail)


def test_preact_follows_the_documented_order():
    """A dense layer equals a plain float32 loop; at p = 0 the head is the eval-mode network."""
    rng = np.random.default_rng(1)
    k, b = rng.normal(size=(6, 4)).astype(np.float32), rng.normal(size=4).astype(np.float32)
    h = rng.normal(size=(3, 6)).astype(np.float32)
    z = MO.preact(h, [(k, b, 0.0, "softmax")], 0, 2)
    for r in range(3):
        want = [np.float32(0)] * 4
        for j in range(6):
            want = [np.float32(want[c] + np.float32(h[r, j] * k[j, c])) for c in range(4)]
        want = [np.float32(want[c] + b[c]) for c in range(4)]
        assert np.array_equal(z[r, 0], np.array(want, dtype=np.float32)) and np.array_equal(z[r, 0], z[r, 1])


def test_head_of_the_case_study_networks():
    first, layers = A.mc_head_layers(mnist.network())
    assert first == 5 and [(l.p, type(l.module).__name__, l.activation) for l in layers] == [(0.5, "Dense", "softmax")]
    first, layers = A.mc_head_layers(imdb.network())
    assert first == 4
    assert [(l.p, l.activation) for l in layers] == [(0.1, "relu"), (0.1, "softmax")]
    assert [tuple(l.module.kernel.shape) for l in layers] == [(32, 20), (20, 2)]


def test_head_of_a_plain_sequential():
    net = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Dropout(0.3), torch.nn.Linear(16, 12),
                              torch.nn.ReLU(), torch.nn.Linear(12, 4), torch.nn.Softmax(dim=1))
    first, layers = A.mc_head_layers(net)
    assert first == 2 and [(l.p, l.activation) for l in layers] == [(0.3, "relu"), (0.0, "softmax")]
    kernel, bias, p, act = A._head_tensors(layers, torch.device("cpu"))[0]
    assert torch.equal(kernel, net[3].weight.t()) and kernel.is_contiguous() and torch.equal(bias, net[3].bias)
    assert A.mc_head_layers(torch.nn.Sequential(torch.nn.Linear(3, 2))) == (-1, [])


@pytest.mark.parametrize("net, match", [
    (lambda: torch.nn.Sequential(torch.nn.Dropout(0.5), torch.nn.Conv2d(1, 2, 3)), "Conv2d"),
    (lambda: torch.nn.Sequential(torch.nn.Dropout(0.5), torch.nn.Linear(4, 2), torch.nn.Softmax(dim=1),
                                 torch.nn.Linear(2, 2)), "softmax"),
    (lambda: torch.nn.Sequential(torch.nn.Dropout(0.5), torch.nn.Dropout(0.5), torch.nn.Linear(4, 2)), "second"),
    (lambda: torch.nn.Sequential(torch.nn.Dropout(0.5), torch.nn.Linear(4, 2), torch.nn.Dropout(0.5)), "end in"),
    (lambda: torch.nn.Sequential(torch.nn.Dropout2d(0.5), torch.nn.Linear(4, 2)), "Dropout2d"),
    (lambda: torch.nn.Sequential(torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.Dropout(0.5)),
                                 torch.nn.Linear(4, 2)), "nested"),
    (lambda: torch.nn.ModuleList([torch.nn.Dropout(0.5), torch.nn.Linear(4, 2)]), "Sequential"),
    (lambda: base.TransformerBlock(8, 2, 8), "Sequential"),
])
def test_heads_it_cannot_sample_are_refused(net, match):
    with pytest.raises(ValueError, match=match):
        A.mc_head_layers(net())


def test_sampler_is_checked_before_any_work():
    with pytest.raises(ValueError, match="sampler"):
        A.get_pred_and_uncertainty(mnist.network(), np.zeros((2, 28, 28, 1), np.float32), sampler="tf")
    with pytest.raises(ValueError, match="Conv2d"):
        A.get_pred_and_uncertainty(torch.nn.Sequential(torch.nn.Dropout(0.5), torch.nn.Conv2d(1, 2, 3)),
                                   np.zeros((2, 1, 5, 5), np.float32), sampler="head")


def test_head_input_must_be_flat_float32_rows():
    assert A.head_input([torch.zeros(3, 4), torch.zeros(2, 4)], 5).shape == (5, 4)
    with pytest.raises(ValueError, match="2-D float32"):
        A.head_input([torch.zeros(3, 4, 2)], 3)
    with pytest.raises(ValueError, match="2-D float32"):
        A.head_input([torch.zeros(3, 4, dtype=torch.float64)], 3)
    with pytest.raises(ValueError, match="rows"):
        A.head_input([torch.zeros(3, 4)], 4)


def _table(*layers):
    keep = [(np.zeros((i, o), np.float32), np.zeros(o, np.float32)) for i, o, _, _ in layers]
    table = (_lib.McLayer * len(layers))()
    for t, ((i, o, p, act), (k, b)) in enumerate(zip(layers, keep)):
        table[t] = _lib.McLayer(k.ctypes.data, b.ctypes.data, p, i, o, act, 0)
    return table, keep


@pytest.mark.parametrize("layers, ok", [
    ([(1600, 10, 0.5, _lib.MC_SOFTMAX)], True),
    ([(32, 20, 0.1, _lib.MC_RELU), (20, 2, 0.1, _lib.MC_SOFTMAX)], True),
    ([(8192, 64, 1.0, _lib.MC_LINEAR)] + [(64, 64, 0.0, _lib.MC_RELU)] * 3, True),
    ([(8193, 10, 0.5, _lib.MC_SOFTMAX)], False),
    ([(16, 65, 0.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 1.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 0.5, _lib.MC_SOFTMAX), (8, 2, 0.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 0.5, _lib.MC_RELU), (9, 2, 0.5, _lib.MC_LINEAR)], False),
    ([(4, 4, 0.0, _lib.MC_RELU)] * 5, False),
])
def test_c_abi_checks_the_head_before_any_launch(layers, ok):
    """rows = 0 returns after the checks, so this runs without a device."""
    table, _keep = _table(*layers)
    out = np.zeros(1, np.float32)
    h = np.zeros(layers[0][0], np.float32)
    rc = _lib.load().tip_mc_head(h.ctypes.data, 0, layers[0][0], 0, 0, 3, table, len(layers), 1, _lib.MC_OUTPUT,
                                 out.ctypes.data, None)
    assert (rc == 0) == ok, _lib.load().tip_last_error()
    assert C.sizeof(_lib.McLayer) == 40      # two pointers, a double, four int32
