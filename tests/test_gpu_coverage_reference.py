"""GPU tests of the coverage kernels (csrc/coverage.cu) against the exact references of oracle/coverage_oracle.py,
through the C ABI, bit for bit (they compute comparisons, counts and an IEEE-sequenced chain):

  * tip_cover_threshold: NAC / SNAC / NBC x the four (activation, boundary) dtype pairs, widths around the 4-neuron,
    128-neuron and 1024-neuron blocks, activation pointers offset by 0, 1 and 4 elements (the float4 and the scalar
    load), values on the boundaries and one ulp either side, +-0, +-inf and NaN activations, NaN and +-inf boundaries,
    profile only / bits only / both; every output starts as 0xAB bytes, so an entry never written shows up;
  * tip_tknc on heavily tied data (small integers, ReLU zeros, +-0, +-inf, NaN) up to 204 800 neurons, k up to d + 5,
    several layers into one profile and one bit set at offsets that are not multiples of 4 or 128;
  * tip_stats_update from arbitrary states and counts (also where float(count) rounds), and the collector over
    ragged badges from NumPy and from CUDA tensors;
  * tip_pack_bool, tip_cam_bits (both gain branches, ties across blocks, continuation across launches), cam /
    cam_from_bits;
  * the classes end to end at CIFAR-like widths and on the reference's own outputs at k <= 0 and non-float NAC inputs.
"""
import time

import numpy as np
import pytest

from oracle import coverage_oracle as CO
from oracle import np_oracle

pytestmark = pytest.mark.gpu

f16, f32, f64 = np.float16, np.float32, np.float64
SENT = 0xABABABAB


def _env():
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    return torch, _lib, _lib.load(), E


def _dev(a):
    torch = _env()[0]
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _words_sentinel(shape):
    return _dev(np.full(shape, SENT, dtype=np.uint32).view(np.int32))


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _offset_view(a, off):
    """a's elements on the device starting `off` elements into an allocation (misaligned for off % 4 != 0)"""
    flat = np.concatenate([np.zeros(off, a.dtype), a.ravel(), np.zeros(4, a.dtype)])
    return _dev(flat)[off:off + a.size]


# ---- tip_cover_threshold -----------------------------------------------------------------------------------------
MODES = {"nac": 0, "snac": 1, "nbc": 2}
NMAX = 3000


def _cover_case(mode, adt, sdt, d, seed):
    rng = np.random.default_rng(seed)
    hi = (rng.normal(size=d) * 2).astype(sdt)
    lo = (hi - np.abs(rng.normal(size=d)) - 0.25).astype(sdt)
    if sdt == f64:
        hi[::2], lo[::2] = hi[::2].astype(f32), lo[::2].astype(f32)     # boundaries a float32 activation can hit
    for arr in (hi, lo):
        arr[rng.random(d) < 0.04] = np.nan
        arr[rng.random(d) < 0.03] = np.inf
        arr[rng.random(d) < 0.03] = -np.inf
    cmp = f32 if (adt, sdt) == (f32, f32) else f64
    thr = cmp(rng.choice([0.3, 0.75, -1.5, 0.0]))
    if mode == "nac":
        b = np.broadcast_to(np.asarray(thr, dtype=sdt), (NMAX, d))
    elif mode == "snac":
        b = np.broadcast_to(hi, (NMAX, d))
    else:
        b = np.where(rng.random((NMAX, d)) < 0.5, lo, hi)
    act = b.astype(adt)                    # on the boundary, unless drawn otherwise below
    kind = rng.integers(0, 20, size=(NMAX, d), dtype=np.int8)
    kind[:, 0] = 0                         # the first neuron of every row sits on its boundary
    for lo_k, hi_k, fill in ((4, 7, lambda v: np.nextafter(v, adt(np.inf))),          # one ulp above
                             (7, 10, lambda v: np.nextafter(v, adt(-np.inf))),        # one ulp below
                             (10, 16, lambda v: rng.normal(size=v.shape) * 2),
                             (16, 17, lambda v: rng.choice(np.array([0.0, -0.0]), size=v.shape)),
                             (17, 18, lambda v: rng.choice(np.array([np.inf, -np.inf]), size=v.shape)),
                             (18, 19, lambda v: np.full(v.shape, np.nan))):
        m = (kind >= lo_k) & (kind < hi_k)
        act[m] = fill(act[m])
    with np.errstate(invalid="ignore"):
        if mode == "nac":
            want = act.astype(cmp) > cmp(thr)
        elif mode == "snac":
            want = act >= hi
        else:
            want = np.stack([act <= lo, act >= hi], axis=2)
    return act, lo, hi, thr, want


def _cover(act_t, adt, n, d, lo_t, hi_t, sdt, thr, mode, want_prof, want_bits):
    torch, _lib, lib, E = _env()
    planes = 2 if mode == "nbc" else 1
    prof = torch.full((n, d * planes), 0xAB, dtype=torch.uint8, device="cuda") if want_prof else None
    bits = _words_sentinel((n, planes * CO.packed_words(d))) if want_bits else None
    score = _words_sentinel((n,))
    _lib.check(lib.tip_cover_threshold(E._p(act_t), E.tip_dtype(adt), n, d, E._p(lo_t), E._p(hi_t), E.tip_dtype(sdt),
                                       float(thr), MODES[mode], E._p(prof), E._p(bits), E._p(score), E._stream()),
               "tip_cover_threshold")
    return (None if prof is None else prof.cpu().numpy()), (None if bits is None else _u32(bits)), score.cpu().numpy()


@pytest.mark.parametrize("d", [1, 3, 4, 5, 31, 127, 128, 129, 1023, 1024, 1025, 4099])
@pytest.mark.parametrize("adt, sdt", [(f32, f32), (f32, f64), (f64, f32), (f64, f64)])
@pytest.mark.parametrize("mode", ["nac", "snac", "nbc"])
def test_cover_threshold_bit_for_bit(mode, adt, sdt, d):
    act, lo, hi, thr, want_all = _cover_case(mode, adt, sdt, d, seed=d * 31 + MODES[mode] * 7 + (adt == f64) * 2 + (sdt == f64))
    planes = 2 if mode == "nbc" else 1
    lo_t = _dev(lo) if mode == "nbc" else None
    hi_t = _dev(hi) if mode != "nac" else None
    for n in (1, 7, NMAX):
        a = np.ascontiguousarray(act[:n])
        want = want_all[:n]
        flat_want = want.reshape(n, d * planes)
        want_score = flat_want.sum(axis=1)
        want_bits = CO.pack_cover(want)                  # padding bits 0
        # offset 0 and 4 elements: the float4 load wherever d % 4 == 0 for float32; offset 1: the scalar load
        for off in ((0, 1) if n == NMAX else (0, 1, 4)):
            at = _offset_view(a, off)
            outs = [(True, True)] if n == NMAX else [(True, False), (False, True), (True, True)]
            for wp, wb in outs:
                where = f"{mode} {np.dtype(adt).name}/{np.dtype(sdt).name} d={d} n={n} off={off} profile={wp} bits={wb}"
                prof, bits, score = _cover(at, adt, n, d, lo_t, hi_t, sdt, thr, mode, wp, wb)
                assert np.array_equal(score, want_score), where
                if wp:
                    assert np.array_equal(prof, flat_want.view(np.uint8)), (where, np.argwhere(prof != flat_want)[:4].tolist())
                if wb:
                    assert np.array_equal(bits, want_bits), (where, np.argwhere(bits != want_bits)[:4].tolist())


# ---- tip_tknc ----------------------------------------------------------------------------------------------------
def _k_for_count(count, d):
    """the reference slice length `count` as the top_neurons argument of tknc_exact"""
    return count if count > 0 else -d


def _tied(rng, n, d, dt):
    x = rng.integers(-2, 3, size=(n, d)).astype(dt)
    relu = np.maximum(rng.normal(size=(n, d)), 0).astype(dt)
    x[1::3] = relu[1::3]                                              # ReLU rows: zeros tie whenever few are positive
    x[2::5] = 0.0                                                     # all-zero rows
    special = rng.random((n, d)) < 0.02
    x[special] = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 0.0], dtype=dt), size=int(special.sum()))
    return x


def _tknc(layers, count, want_prof=True, want_bits=True):
    torch, _lib, lib, E = _env()
    n = layers[0].shape[0]
    total = sum(l.shape[1] for l in layers)
    words = CO.packed_words(total)
    prof = torch.full((n, total), 0xAB, dtype=torch.uint8, device="cuda") if want_prof else None
    bits = torch.zeros((n, words), dtype=torch.int32, device="cuda") if want_bits else None
    off = 0
    for l in layers:
        lt = _dev(l)
        _lib.check(lib.tip_tknc(E._p(lt), E.tip_dtype(l.dtype), n, l.shape[1], count, E._p(prof), total, off, E._p(bits),
                                words, E._stream()), "tip_tknc")
        off += l.shape[1]
    return (None if prof is None else prof.cpu().numpy()), (None if bits is None else _u32(bits))


@pytest.mark.parametrize("d", [1, 2, 255, 256, 257, 4097, 49153, 204800])
@pytest.mark.parametrize("dt", [f32, f64])
def test_tknc_bit_for_bit(dt, d):
    rng = np.random.default_rng(d + (dt == f64))
    n = 40 if d <= 4097 else (5 if d <= 49153 else 2)
    x = _tied(rng, n, d, dt)
    counts = [1, 3, d - 1, d, d + 5] if d <= 4097 else [1, 3, d, d + 5]
    for k in sorted(set(c for c in counts if c >= 0)):
        where = f"{np.dtype(dt).name} d={d} k={k}"
        prof, bits = _tknc([x], k)
        want = CO.tknc_exact(_k_for_count(k, d), [x])[1]
        assert np.array_equal(prof, want.astype(np.uint8)), (where, np.argwhere(prof != want)[:4].tolist())
        assert np.array_equal(CO.unpack_cover(bits, d), want), where
        assert np.array_equal(CO.pack_cover(want), bits), where
        assert np.all(want.sum(axis=1) == min(k, d)), where


def test_tknc_layers_into_one_profile_at_odd_offsets():
    rng = np.random.default_rng(5)
    widths = [5, 131, 1, 257, 4097]                                    # offsets 0, 5, 136, 137, 394
    layers = [_tied(rng, 30, w, f32 if i % 2 == 0 else f64) for i, w in enumerate(widths)]
    total = sum(widths)
    for k in (1, 3, 6):
        prof, bits = _tknc(layers, k)
        want = CO.tknc_exact(k, layers)[1]
        assert np.array_equal(prof, want.astype(np.uint8)), k
        assert np.array_equal(CO.unpack_cover(bits, total), want) and np.array_equal(CO.pack_cover(want), bits), k
        only_bits = _tknc(layers, k, want_prof=False)[1]
        only_prof = _tknc(layers, k, want_bits=False)[0]
        assert np.array_equal(only_bits, bits) and np.array_equal(only_prof, prof), k


def test_tknc_rejects_layers_past_the_shared_memory_flags():
    torch, _lib, lib, E = _env()
    x = torch.zeros((1, 204801), dtype=torch.float32, device="cuda")
    prof = torch.zeros((1, 204801), dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.TipError):
        _lib.check(lib.tip_tknc(E._p(x), _lib.TIP_F32, 1, 204801, 1, E._p(prof), 204801, 0, None, 0, E._stream()), "tip_tknc")


# ---- tip_stats_update --------------------------------------------------------------------------------------------
def _bits_equal(a, b):
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("count", [0, 1, 5, 2 ** 24 - 3, 2 ** 24 + 1])
@pytest.mark.parametrize("dt", [f32, f64])
def test_stats_update_bit_for_bit(dt, count):
    torch, _lib, lib, E = _env()
    rng = np.random.default_rng(count % 977 + 3 * (dt == f64))
    for d in (1, 127, 128, 129, 1000):
        for n in (1, 7, 8, 9, 23):
            x = (rng.normal(size=(n, d)) * 3).astype(dt)
            mean = rng.normal(size=d).astype(dt)
            mean[::3] = 0                                  # the whole new mean is delta / count: its rounding shows
            state = [mean, (rng.random(d) * 5).astype(dt), (mean - rng.random(d)).astype(dt), (mean + rng.random(d)).astype(dt)]
            if count == 0 and n == 7:
                state = [np.zeros(d, dt), np.zeros(d, dt), np.full(d, np.inf, dt), np.full(d, -np.inf, dt)]   # a fresh fit
            dev = [_dev(s.copy()) for s in state]
            _lib.check(lib.tip_stats_update(E._p(_dev(x)), E.tip_dtype(dt), n, d, count, *(E._p(t) for t in dev),
                                            E._stream()), "tip_stats_update")
            want = CO.welford_from(x, count, *state)
            for name, g, w in zip(("mean", "m2", "min", "max"), dev, want):
                assert _bits_equal(g.cpu().numpy(), w), (np.dtype(dt).name, count, d, n, name)


@pytest.mark.parametrize("from_device", [False, True])
def test_collector_over_ragged_badges(from_device):
    torch = _env()[0]
    from simple_tip_b200.core.aggregate_statistics import AggregateStatisticsCollector
    from simple_tip_b200.core.neuron_coverage import NBC

    rng = np.random.default_rng(61)
    shapes = [(4, 3, 5), (129,), (1,)]
    sizes = [1, 7, 8, 9, 33]
    data = [np.maximum(rng.normal(size=(sum(sizes),) + sh) * 2 + 0.3, 0).astype(f32) for sh in shapes]
    data[1] = data[1].astype(f64)
    cuts = np.cumsum([0] + sizes)
    badges = [[l[a:b] for l in data] for a, b in zip(cuts[:-1], cuts[1:])]
    wrap = (lambda a: torch.from_numpy(a).cuda()) if from_device else (lambda a: a)
    col = AggregateStatisticsCollector()
    for badge in badges:
        col.track([wrap(l) for l in badge])
    got = col.get()
    want = np_oracle.stats_oracle(badges)
    for gl, wl in zip(got, want):
        for g, w in zip(gl, wl):
            assert g.shape == w.shape and _bits_equal(g, w)
    # one sample: std is NaN, so every NBC boundary is NaN and nothing is covered (as in the reference)
    one = AggregateStatisticsCollector()
    one.track([wrap(l[:1]) for l in data])
    mins, maxs, stds = one.get()
    assert all(np.isnan(s).all() for s in stds)
    test = [l[:6] for l in data]
    score, prof = NBC(mins, maxs, stds, 0.5)(test)
    ws, wp = np_oracle.nbc_oracle(mins, maxs, stds, 0.5, test)
    assert not wp.any() and np.array_equal(prof, wp) and score.dtype == ws.dtype and np.array_equal(score, ws)


def test_collector_runs_float16_badges_in_float32():
    """A documented deviation: float16 badges are folded in float32 (the reference keeps float16 arithmetic)."""
    from simple_tip_b200.core.aggregate_statistics import AggregateStatisticsCollector

    rng = np.random.default_rng(62)
    x = rng.normal(size=(20, 50)).astype(f16)
    col = AggregateStatisticsCollector()
    col.track([x[:9]])
    col.track([x[9:]])
    got = col.get()
    want = np_oracle.stats_oracle([[x[:9].astype(f32)], [x[9:].astype(f32)]])
    assert all(_bits_equal(g[0], w[0]) for g, w in zip(got, want))


# ---- tip_pack_bool -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [1, 31, 32, 33, 1000])
def test_pack_bool_bit_for_bit(f):
    torch, _lib, lib, E = _env()
    rng = np.random.default_rng(f)
    prof = rng.choice(np.array([0, 1, 2, 255], dtype=np.uint8), size=(9, f))
    prof[0] = 0
    prof[1] = 2                                                     # every byte value other than 0 counts as covered
    bits = _words_sentinel((9, -(-f // 32)))
    _lib.check(lib.tip_pack_bool(E._p(_dev(prof)), 9, f, E._p(bits), E._stream()), "tip_pack_bool")
    assert np.array_equal(_u32(bits), CO.pack_plain(prof))
    from simple_tip_b200.core.prioritizers import pack_profiles

    assert np.array_equal(_u32(pack_profiles(prof != 0)), CO.pack_plain(prof))


# ---- tip_cam_bits ------------------------------------------------------------------------------------------------
def _cam_greedy_gpu(prof, rounds):
    """the greedy picks and the final state[0] of tip_cam_bits, called until it is done, as cam_from_bits does"""
    torch, _lib, lib, E = _env()
    n = prof.shape[0]
    bits = _dev(CO.pack_plain(prof).view(np.int32))
    words = bits.shape[1]
    gain = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    covered = torch.zeros(2 * words, dtype=torch.int32, device="cuda")
    cand = torch.zeros(4 * _lib.CAM_MAX_BLOCKS, dtype=torch.int32, device="cuda")
    order = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    state = torch.zeros(4, dtype=torch.int32, device="cuda")
    picks, done, first, launches = 0, False, 1, 0
    while not done and picks < n:
        _lib.check(lib.tip_cam_bits(E._p(bits), n, words, E._p(gain), E._p(covered), E._p(cand), E._p(order), E._p(state),
                                    rounds, first, E._stream()), "tip_cam_bits")
        first, launches = 0, launches + 1
        st = state.cpu().numpy()
        picks, done = int(st[0]), bool(st[1])
    return order.cpu().numpy()[:picks].astype(np.int64), launches


def _cam_profiles():
    rng = np.random.default_rng(71)
    out = {"n1": rng.random((1, 70)) < 0.3}
    p = rng.random((50, 200)) < 0.05
    p[[9, 30, 44]] = rng.random(200) < 0.5                           # duplicate best rows
    p[::7] = False                                                   # all-zero rows
    out["n50"] = p
    early = rng.random((50, 96)) < 0.05
    early[17] = True                                                 # covers everything with the first pick
    out["n50_early"] = early
    big = rng.random((20000, 640)) < 0.004
    # equal gains on disjoint entries in different blocks' slices (the grid is 2 blocks per SM, ~76 rows each):
    # the lowest index must win every time across blocks
    for j, r in enumerate([19990, 12000, 7000, 77, 3]):
        big[r] = False
        big[r, 100 * j:100 * j + 60] = True
    big[[15000, 401]] = big[77]                                     # and identical copies of one of them
    out["n20000"] = big
    # 160 000 entries (5000 words): the first pick covers 31 bits of 4500 words, the second then has 5000 > 4096 fresh
    # words (the dense-pick branch, with entries already covered), later picks fewer (the listed-word branch)
    dense = rng.random((300, 160000)) < 0.005
    w = np.arange(160000) // 32
    b = np.arange(160000) % 32
    dense[11] = (w < 4500) & (b != 0)
    dense[200] = (b == 0) | ((b == 1) & (w < 4800))
    out["dense"] = dense
    return out


@pytest.mark.parametrize("case", ["n1", "n50", "n50_early", "n20000", "dense"])
def test_cam_bits_greedy_and_order(case):
    from simple_tip_b200.core.prioritizers import cam, cam_from_bits

    prof = _cam_profiles()[case]
    want_greedy = CO.cam_greedy(prof)
    score = prof.sum(axis=1)
    want = np_oracle.cam_oracle(score, prof)
    if case == "dense":
        assert list(want_greedy[:2]) == [11, 200]
    results = []
    for rounds in (2, 4, 4096):
        greedy, launches = _cam_greedy_gpu(prof, rounds)
        assert np.array_equal(greedy, want_greedy), (case, rounds, greedy[:8].tolist(), want_greedy[:8].tolist())
        if rounds == 2 and want_greedy.shape[0] > 2:
            assert launches > 1                                      # the loop continued across launches
        bits = _dev(CO.pack_plain(prof).view(np.int32))
        results.append(np.array(list(cam_from_bits(score, bits, rounds_per_launch=rounds))))
        assert np.array_equal(results[-1], want), (case, rounds)
    assert np.array_equal(np.array(list(cam(score, prof))), want), case


# ---- the classes end to end ---------------------------------------------------------------------------------------
CIFAR = [(32, 32, 64), (16, 16, 64), (8, 8, 128)]                   # 65 536 + 16 384 + 8 192 neurons


def test_classes_at_cifar_widths_in_mixed_dtypes():
    torch = _env()[0]
    from simple_tip_b200.core.neuron_coverage import NAC, NBC, SNAC, TKNC
    from simple_tip_b200.core.prioritizers import cam_from_bits

    rng = np.random.default_rng(81)
    n = 24
    train = [np.maximum(rng.normal(size=(64,) + sh) + 0.1, 0).astype(f64) for sh in CIFAR]
    mins = [l.min(axis=0) for l in train]
    maxs = [l.max(axis=0) for l in train]
    stds = [l.std(axis=0) for l in train]
    test = [np.maximum(rng.normal(size=(n,) + sh) * 1.3 + 0.1, 0).astype(f32) for sh in CIFAR]
    test[0][0, :2] = maxs[0][:2].astype(f32)
    half = [l.astype(f16) for l in test]
    cases = {
        "NAC_f16": (NAC(0.3), half, lambda: np_oracle.nac_oracle(0.3, half)),
        "NAC_f32": (NAC(0.75), test, lambda: np_oracle.nac_oracle(0.75, test)),
        "SNAC_f32_f64": (SNAC(maxs, stds, 0.5), test, lambda: np_oracle.snac_oracle(maxs, stds, 0.5, test)),
        "NBC_f32_f64": (NBC(mins, maxs, stds, 0.5), test, lambda: np_oracle.nbc_oracle(mins, maxs, stds, 0.5, test)),
        "NBC_f16_f64": (NBC(mins, maxs, stds, 0), half, lambda: np_oracle.nbc_oracle(mins, maxs, stds, 0, half)),
    }
    mixed = [test[0], test[1].astype(f64), half[2]]
    for k in (1, 3, 0):
        cases[f"TKNC_{k}"] = (TKNC(k), mixed, lambda k=k: CO.tknc_exact(k, mixed))
    for name, (metric, acts, oracle) in cases.items():
        ws, wp = oracle()
        gs, gp = metric([l.copy() for l in acts])
        assert gs.dtype == ws.dtype and np.array_equal(gs, ws), name
        assert gp.shape == wp.shape and np.array_equal(gp, wp), name
        ps, bits = metric.packed([torch.from_numpy(l).cuda() for l in acts])
        planes = 2 if wp.ndim == 3 else 1
        d = wp.shape[1]
        assert np.array_equal(ps.cpu().numpy(), ws.astype(np.int32)), name
        assert np.array_equal(CO.unpack_cover(_u32(bits), d, planes), wp), name
        assert np.array_equal(np.array(list(cam_from_bits(ws, bits))), np_oracle.cam_oracle(ws, wp)), name


def test_classes_reproduce_the_reference_at_k_le_0_and_non_float_nac(golden):
    torch = _env()[0]
    from simple_tip_b200.core.neuron_coverage import NAC, TKNC

    g = golden("coverage_edges_reference.npz")
    layers = [g[f"tknc.layer{i}"] for i in range(3)]
    d = sum(l.shape[1] for l in layers)
    for k in (0, -1, -3, d, d + 2):
        score, prof = TKNC(k)([l.copy() for l in layers])
        want_s, want_p = g[f"tknc.k{k}.score"], g[f"tknc.k{k}.profile"]
        assert score.dtype == want_s.dtype and np.array_equal(score, want_s), k
        assert np.array_equal(prof, want_p), k
        ps, bits = TKNC(k).packed([torch.from_numpy(l).cuda() for l in layers])
        assert np.array_equal(ps.cpu().numpy(), want_s.astype(np.int32)) and np.array_equal(CO.unpack_cover(_u32(bits), d), want_p), k
    for name in ("f16", "i16", "u8", "bool"):
        act = g[f"nac.{name}.act"]
        for t in (0.3, 0.75, 0.9999999999, 1.9999999999):
            want_s, want_p = g[f"nac.{name}.{t!r}.score"], g[f"nac.{name}.{t!r}.profile"]
            score, prof = NAC(t)([act.copy()])
            assert score.dtype == want_s.dtype and np.array_equal(score, want_s), (name, t)
            assert np.array_equal(prof, want_p), (name, t)
            ps, bits = NAC(t).packed([torch.from_numpy(act).cuda()])          # torch tensors follow NumPy's dtype
            assert np.array_equal(ps.cpu().numpy(), want_s.astype(np.int32)), (name, t)
            assert np.array_equal(CO.unpack_cover(_u32(bits), act.shape[1]), want_p), (name, t)


def test_tknc_count_short_circuit_is_quick_on_a_wide_layer():
    """TKNC(0) marks every neuron without running one selection round per neuron (21 632 neurons: an MNIST conv)."""
    import torch

    from simple_tip_b200.core.neuron_coverage import TKNC

    x = torch.from_numpy(np.random.default_rng(9).normal(size=(256, 21632)).astype(f32)).cuda()
    TKNC(0).packed([x])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    score, bits = TKNC(0).packed([x])
    torch.cuda.synchronize()
    assert time.perf_counter() - t0 < 1.0
    assert np.all(score.cpu().numpy() == 21632) and CO.unpack_cover(_u32(bits), 21632).all()
