"""Pins oracle/coverage_oracle.py, the exact references of the coverage kernels (csrc/coverage.cu), against the
reference's own TKNC / NAC (tests/golden/coverage_edges_reference.npz, oracle/make_golden.py: coverage_edge_cases),
against np_oracle on tie-free data, and against brute-force restatements of each rule.  Each comparison is also run
with a defect injected into the oracle (layout, tie rule, count dtype, CAM tie rule) and must then fail."""
import numpy as np
import pytest

from oracle import coverage_oracle as CO
from oracle import np_oracle
from oracle.ref_harness import Welford025

f16, f32, f64 = np.float16, np.float32, np.float64


# ---- defects -----------------------------------------------------------------------------------------------------
def _grid_swapped(a):
    n, w = a.shape
    return a.reshape(n, w // 128, 4, 32).transpose(0, 1, 3, 2)       # neuron 128g + 32i + l


def _top_order_ties_low(flat):
    d = flat.shape[1]
    return (d - 1 - np.argsort(flat[:, ::-1], axis=1, kind="stable"))   # equal values: the LOWER index ranks higher


def _count_f64(t, count):
    return np.float64(count)


def _last_argmax(gain):
    return int(gain.shape[0] - 1 - np.argmax(gain[::-1]))


# ---- layouts -----------------------------------------------------------------------------------------------------
def _layout_known_answer(d):
    """Every single-neuron profile lands in word 4*(c // 128) + c % 4, bit (c % 128) // 4."""
    prof = np.eye(d, dtype=bool)
    bits = CO.pack_cover(prof)
    want = np.zeros((d, CO.packed_words(d)), dtype=np.uint32)
    c = np.arange(d)
    want[c, 4 * (c // 128) + c % 4] = np.left_shift(np.uint32(1), ((c % 128) // 4).astype(np.uint32))
    return np.array_equal(bits, want)


@pytest.mark.parametrize("d", [1, 3, 4, 5, 127, 128, 129, 300])
def test_pack_cover_layout_and_round_trip(d):
    assert _layout_known_answer(d)
    rng = np.random.default_rng(d)
    prof = rng.random((7, d)) < 0.4
    bits = CO.pack_cover(prof)
    assert bits.dtype == np.uint32 and bits.shape == (7, CO.packed_words(d))
    assert np.array_equal(CO.unpack_cover(bits, d), prof)
    assert np.array_equal(CO.unpack_cover(bits.view(np.int32), d), prof)       # as torch hands int32 words back
    two = rng.random((7, d, 2)) < 0.4                                          # NBC: lower plane first
    b2 = CO.pack_cover(two)
    assert np.array_equal(b2[:, :CO.packed_words(d)], CO.pack_cover(two[..., 0]))
    assert np.array_equal(CO.unpack_cover(b2, d, planes=2), two)
    # a set padding bit does not survive the round trip
    if d % 128:
        bad = bits.copy()
        c = d                                                                  # the first padding neuron
        bad[0, 4 * (c // 128) + c % 4] |= np.uint32(1) << np.uint32((c % 128) // 4)
        assert not np.array_equal(CO.pack_cover(CO.unpack_cover(bad, d)), bad)


def test_pack_cover_rejects_swapped_layout(monkeypatch):
    monkeypatch.setattr(CO, "_grid", _grid_swapped)
    prof = np.random.default_rng(0).random((5, 300)) < 0.5
    assert np.array_equal(CO.unpack_cover(CO.pack_cover(prof), 300), prof)     # still its own inverse ...
    assert not _layout_known_answer(300)                                       # ... but not the kernel's layout


@pytest.mark.parametrize("f", [1, 31, 32, 33, 1000])
def test_pack_plain_layout(f):
    rng = np.random.default_rng(f)
    prof = rng.choice(np.array([0, 1, 2, 255], dtype=np.uint8), size=(4, f))
    bits = CO.pack_plain(prof)
    assert bits.shape == (4, -(-f // 32))
    for r in range(4):
        for e in range(f):
            assert bool((int(bits[r, e // 32]) >> (e % 32)) & 1) == bool(prof[r, e])
    pad = np.zeros((4, 32 * bits.shape[1]), dtype=bool)
    pad[:, :f] = prof != 0
    assert np.array_equal(np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little").astype(bool), pad)


# ---- TKNC --------------------------------------------------------------------------------------------------------
def _tknc_bruteforce(k, layers):
    """neuron i is marked iff fewer than len(range(d)[-k:]) neurons rank above it; j ranks above i when x_j > x_i, or
    x_j == x_i and j > i; NaN ranks above every number, and NaNs among themselves by index"""
    out = []
    for layer in layers:
        x = layer.reshape(layer.shape[0], -1).astype(f64)
        n, d = x.shape
        cnt = len(range(d)[-k:])
        mark = np.zeros((n, d), dtype=bool)
        j = np.arange(d)
        for r in range(n):
            v = x[r]
            nan = np.isnan(v)
            for i in range(d):
                if nan[i]:
                    above = nan & (j > i)
                else:
                    above = nan | (v > v[i]) | ((v == v[i]) & (j > i))
                mark[r, i] = above.sum() < cnt
        out.append(mark)
    return np.concatenate(out, axis=1)


def _tied_layers(rng):
    a = rng.integers(0, 3, size=(6, 17)).astype(f32)              # small integers
    b = np.maximum(rng.normal(size=(6, 2, 5)), 0).astype(f32)      # ReLU zeros
    b[0] = 0.0
    c = rng.integers(-2, 2, size=(6, 9)).astype(f64)
    c[1, 3], c[1, 5], c[2, 0], c[3, 1], c[3, 2] = np.nan, np.nan, np.inf, -np.inf, -0.0
    c[4, :4] = [0.0, -0.0, 0.0, -0.0]
    return [a, b, c]


def test_tknc_exact_matches_reference_golden(golden):
    g = golden("coverage_edges_reference.npz")
    layers = [g[f"tknc.layer{i}"] for i in range(3)]
    d = sum(l.shape[1] for l in layers)
    for k in (0, -1, -3, d, d + 2):
        score, prof = CO.tknc_exact(k, layers)
        want_s, want_p = g[f"tknc.k{k}.score"], g[f"tknc.k{k}.profile"]
        assert score.dtype == want_s.dtype and np.array_equal(score, want_s), k
        assert np.array_equal(prof, want_p), k
        assert np.all(score == sum(CO.tknc_count(k, l.shape[1]) for l in layers)), k
    assert np.all(g["tknc.k0.score"] == d) and np.all(g["tknc.k-1.score"] == d - 3)     # the width-1 layer marks nothing


def test_tknc_exact_matches_np_oracle_on_tie_free_data():
    rng = np.random.default_rng(3)
    layers = [rng.normal(size=(20, 37)).astype(f32), rng.normal(size=(20, 3, 4)), rng.normal(size=(20, 1)).astype(f32)]
    for k in (-40, -2, -1, 0, 1, 2, 3, 12, 36, 37, 38, 100):
        ws, wp = np_oracle.tknc_oracle(k, layers)
        gs, gp = CO.tknc_exact(k, layers)
        assert gs.dtype == ws.dtype and np.array_equal(gs, ws) and np.array_equal(gp, wp), k


@pytest.mark.parametrize("k", [-4, -1, 0, 1, 3, 8, 17, 30])
def test_tknc_exact_tie_rule_matches_bruteforce(k):
    layers = _tied_layers(np.random.default_rng(k + 50))
    assert np.array_equal(CO.tknc_exact(k, layers)[1], _tknc_bruteforce(k, layers)), k


def test_tknc_bruteforce_rejects_inverted_tie_rule(monkeypatch):
    layers = _tied_layers(np.random.default_rng(7))
    monkeypatch.setattr(CO, "_top_order", _top_order_ties_low)
    assert any(not np.array_equal(CO.tknc_exact(k, layers)[1], _tknc_bruteforce(k, layers)) for k in (1, 3, 8))


# ---- NAC ---------------------------------------------------------------------------------------------------------
def test_nac_golden_is_numpys_own_promotion(golden):
    """The reference's NAC on float16 / integer / bool activations is `act > t` in NumPy's promoted dtype; the
    float32 comparison the classes used before differs on these cases (which is what the golden file pins)."""
    g = golden("coverage_edges_reference.npz")
    differs = set()
    for name in ("f16", "i16", "u8", "bool"):
        act = g[f"nac.{name}.act"]
        for t in (0.3, 0.75, 0.9999999999, 1.9999999999):
            want = g[f"nac.{name}.{t!r}.profile"]
            assert np.array_equal(act > t, want)
            cmp = np.result_type(act.dtype, t)
            assert np.array_equal(act.astype(f64) > np.asarray(t).astype(cmp).astype(f64), want)
            if not np.array_equal(act.astype(f32) > f32(t), want):
                differs.add(name)
    assert differs == {"f16", "i16", "u8", "bool"}


# ---- Welford -----------------------------------------------------------------------------------------------------
def _literal_welford(x, count, mean, m2, mn, mx):
    """welford==0.2.5's add_all on a Welford restored to the given state (its in-place NumPy expressions with a
    Python-int count) plus np.minimum / np.maximum"""
    w = Welford025()
    w._shape, w._count, w._m, w._s = mean.shape, count, mean.copy(), m2.copy()
    w.add_all(x)
    return w._m, w._s, np.minimum(mn, x.min(axis=0)), np.maximum(mx, x.max(axis=0))


def _state(rng, d, dt):
    mean = rng.normal(size=d).astype(dt)
    mean[::3] = 0          # the quotient delta / count is the whole new mean: its rounding shows at any count
    return mean, (rng.random(d) * 3).astype(dt), (mean - 1).astype(dt), (mean + 1).astype(dt)


def _same_bits(a, b):
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("count", [0, 1, 5, 2 ** 24 - 3, 2 ** 24 + 1])
def test_welford_from_matches_literal_welford(dt, count):
    rng = np.random.default_rng(count % 1000 + (dt == f64))
    x = (rng.normal(size=(9, 40)) * 4).astype(dt)
    state = _state(rng, 40, dt)
    got = CO.welford_from(x, count, *state)
    want = _literal_welford(x, count, *state)
    for a, b in zip(got, want):
        assert _same_bits(a, b), (dt, count)


def test_welford_from_empty_state_matches_stats_oracle():
    rng = np.random.default_rng(11)
    x = (rng.normal(size=(23, 30)) * 2).astype(f32)
    mean, m2, mn, mx = CO.welford_from(x, 0, np.zeros(30, f32), np.zeros(30, f32), np.full(30, np.inf, f32),
                                       np.full(30, -np.inf, f32))
    o_min, o_max, o_std = np_oracle.stats_oracle([[x[:8]], [x[8:]]])
    assert np.array_equal(mn, o_min[0]) and np.array_equal(mx, o_max[0])
    assert np.array_equal(np.sqrt(m2 / (23 - 1)), o_std[0])


def test_welford_rejects_count_divided_in_float64(monkeypatch):
    """(float)count rounds at 2^24 + 1: NumPy divides by float32(count), which a float64 division does not"""
    rng = np.random.default_rng(12)
    x = (rng.normal(size=(4, 200)) * 4).astype(f32)
    state = _state(rng, 200, f32)
    want = _literal_welford(x, 2 ** 24 + 1, *state)
    monkeypatch.setattr(CO, "_count_as", _count_f64)
    got = CO.welford_from(x, 2 ** 24 + 1, *state)
    assert not all(_same_bits(a, b) for a, b in zip(got[:2], want[:2]))


# ---- CAM ---------------------------------------------------------------------------------------------------------
def _cam_cases():
    rng = np.random.default_rng(21)
    dup = rng.random((60, 90)) < 0.1
    dup[[7, 33, 51]] = rng.random(90) < 0.6                  # three identical best rows
    zero = rng.random((30, 40)) < 0.2
    zero[::3] = False                                        # all-zero rows
    early = rng.random((40, 64)) < 0.05
    early[5] = True                                          # one row covers everything at once
    return [dup, zero, early, rng.random((200, 300)) < 0.03, np.zeros((4, 10), dtype=bool)]


def test_cam_greedy_is_the_head_of_cam_oracle(golden):
    for prof in _cam_cases():
        greedy = CO.cam_greedy(prof)
        full = np_oracle.cam_oracle(prof.sum(axis=1), prof)
        assert np.array_equal(full[:greedy.shape[0]], greedy)
        assert not prof.any() or greedy.shape[0] >= 1
        covered = np.zeros(prof.shape[1], dtype=bool)
        for i in greedy:
            assert (prof[i] & ~covered).any()                # every pick covers something new
            covered |= prof[i]
        assert np.array_equal(covered, prof.any(axis=0))     # and together they cover everything coverable
    g = golden("prioritizers_reference.npz")
    for i in range(4):
        prof, order = g[f"cam{i}.profiles"], g[f"cam{i}.order"]
        greedy = CO.cam_greedy(prof)
        assert np.array_equal(order[:greedy.shape[0]], greedy), i


def test_cam_greedy_rejects_ties_to_the_highest_index(monkeypatch):
    prof = _cam_cases()[0]
    want = np_oracle.cam_oracle(prof.sum(axis=1), prof)
    monkeypatch.setattr(CO, "_first_argmax", _last_argmax)
    greedy = CO.cam_greedy(prof)
    assert not np.array_equal(want[:greedy.shape[0]], greedy)
