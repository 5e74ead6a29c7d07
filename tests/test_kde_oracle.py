"""CPU tests of the float64 references of the LSA kernels (oracle/kde_oracle.py) that the device pass is compared
against: the packing emulations against torch's bfloat16 / float16 conversions, the partials against
scipy.special.logsumexp, the premise of the exact construction, the power of the exact comparison (each kernel defect
below is rejected), the work-list checker, the merge references, and the host side of the density: the underflow rule
of StableGaussianKDE._finish."""
import math

import numpy as np
import pytest
import torch
from scipy.special import logsumexp

from oracle import kde_oracle as KO
from oracle import sil_oracle as SO
from simple_tip_b200 import engine as E

f32, f64 = np.float32, np.float64


def _torch_round(v, dtype):
    """float32 values rounded by torch's own conversion, returned as float32"""
    return torch.from_numpy(np.ascontiguousarray(v, dtype=f32)).to(dtype).to(torch.float32).numpy()


# ---- packing ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [f32, f64])
@pytest.mark.parametrize("d", [1, 15, 16, 17, 97])
def test_pack_lse_matches_torch_bfloat16(d, dtype):
    rng = np.random.default_rng(d + 100 * (dtype == f64))
    x = (rng.normal(size=(64, d)) * np.exp(rng.normal(size=(64, 1)) * 3)).astype(dtype)
    x[3] = 0.0
    center = rng.normal(size=d).astype(f32)
    d16 = -(-d // 16) * 16
    for cen in (None, center):
        v = (x - (0 if cen is None else cen)).astype(f32) if dtype == f32 else \
            (x - (0.0 if cen is None else cen.astype(f64))).astype(f32)
        h = _torch_round(v, torch.bfloat16)
        lo = _torch_round(v - h, torch.bfloat16)
        sq = np.sum(v.astype(f64) ** 2, axis=1).astype(f32)
        q, qsq = KO.pack_lse(x, "query", cen)
        t, tsq = KO.pack_lse(x, "train", cen)
        assert q.shape == t.shape == (64, SO.pair_pitch(d))
        assert np.array_equal(qsq, sq) and np.array_equal(tsq, sq)
        qv, tv = KO.decode(q, "bf16"), KO.decode(t, "bf16")
        for seg, (want_q, want_t) in enumerate(((h, h), (lo, h), (h, lo))):
            assert np.array_equal(qv[:, seg * d16:seg * d16 + d], want_q)
            assert np.array_equal(tv[:, seg * d16:seg * d16 + d], want_t)
            assert not np.any(qv[:, seg * d16 + d:(seg + 1) * d16]) and not np.any(tv[:, seg * d16 + d:(seg + 1) * d16])
        c = np.float32(-0.5) * sq
        c0 = _torch_round(c, torch.bfloat16)
        c1 = _torch_round(c - c0, torch.bfloat16)
        c2 = _torch_round((c - c0) - c1, torch.bfloat16)
        assert np.array_equal(tv[:, 3 * d16:3 * d16 + 3], np.stack([c0, c1, c2], axis=1))
        assert np.all(qv[:, 3 * d16:3 * d16 + 3] == 1.0)
        assert not np.any(qv[:, 3 * d16 + 3:]) and not np.any(tv[:, 3 * d16 + 3:])


@pytest.mark.parametrize("dtype", [f32, f64])
@pytest.mark.parametrize("d", [1, 16, 17, 305])
def test_pack_f16_matches_torch_float16(d, dtype):
    rng = np.random.default_rng(d + 7)
    x = (rng.normal(size=(64, d)) * np.exp(rng.normal(size=(64, 1)) * 3)).astype(dtype)
    x = np.clip(x, -6e4, 6e4)
    x[2] = 0.0
    x[4, 0] = 3.0e-6                    # an fp16 subnormal
    d16 = -(-d // 16) * 16
    for role in ("query", "train"):
        pk, sq, _ = KO.pack_f16(x, role, -0.5 if role == "train" else 0.0, 64.0)
        v = x.astype(f32)
        val = KO.decode(pk, "f16")
        assert pk.shape == (64, KO.pair_pitch1(d))
        assert np.array_equal(val[:, :d], _torch_round(v, torch.float16))
        assert np.array_equal(val[:, :d], v.astype(np.float16).astype(f64))
        assert not np.any(val[:, d:d16]) and not np.any(val[:, d16 + 3:])
        assert np.array_equal(sq, np.sum(v.astype(f64) ** 2, axis=1).astype(f32))
        if role == "query":
            assert np.all(val[:, d16:d16 + 3] == 64.0)
        else:
            cv = (np.float32(-0.5) * sq) / np.float32(64.0)
            c0 = _torch_round(cv, torch.float16)
            c1 = _torch_round(cv - c0, torch.float16)
            with np.errstate(invalid="ignore"):          # rows whose norm term overflows: inf, then NaN
                c2 = _torch_round((cv - c0) - c1, torch.float16)
            assert np.array_equal(val[:, d16:d16 + 3], np.stack([c0, c1, c2], axis=1), equal_nan=True)


def test_pack_f16_flags():
    """65504 is fp16's largest finite value: it does not raise the flag in the query role; 65520 (rounds to inf), inf
    and NaN do; a train row raises it when -|v|^2 / 2 / S leaves the range (S = 64: |v|^2 > 8 384 512)"""
    flag = lambda rows, role: KO.pack_f16(np.asarray(rows, dtype=f32), role, -0.5 if role == "train" else 0.0, 64.0)[2]
    assert not flag([[65504.0, -65504.0]], "query")
    for bad in (65520.0, -65520.0, np.inf, np.nan):
        assert flag([[1.0, bad]], "query") and flag([[1.0, bad]], "train")
    assert flag([[65504.0]], "train")                 # its norm term is far out of range
    assert flag([[2896.0, 0.0]], "train") and not flag([[2896.0, 0.0]], "query")
    assert not flag([[2895.0, 0.0]], "train")


# ---- float64 partials ------------------------------------------------------------------------------------------
def test_lse_parts_matches_scipy_logsumexp():
    rng = np.random.default_rng(11)
    m, n, d = 70, 700, 20
    x = rng.normal(size=(m, d)) * 2.0
    y = rng.normal(size=(n, d))
    q, _ = KO.pack_lse(x.astype(f32), "query")
    t, _ = KO.pack_lse(y.astype(f32), "train")
    items, slots = E.build_items(np.array([0, m]), [[(0, n)]], 1)
    pm, ps, cov = KO.lse_parts(q, t, items, slots, m)
    assert cov.all()
    # an independent decode: torch's bfloat16 -> float64, and a NumPy product
    qd = torch.from_numpy(q.view(np.int16)).view(torch.bfloat16).to(torch.float64).numpy()
    td = torch.from_numpy(t.view(np.int16)).view(torch.bfloat16).to(torch.float64).numpy()
    a = qd @ td.T
    for q0, qr, c0, c1, s, _ in items.tolist():
        blk = a[q0:q0 + qr, c0:c1]
        assert np.allclose(pm[s, q0:q0 + qr], blk.max(1), rtol=0, atol=1e-12)
        lse = logsumexp(blk, axis=1)
        assert np.allclose(pm[s, q0:q0 + qr] + np.log(ps[s, q0:q0 + qr]), lse, rtol=1e-14, atol=1e-12)
    # fp16 operands the same way
    qf, _, _ = KO.pack_f16(x.astype(f32), "query", 0.0, 64.0)
    tf, _, _ = KO.pack_f16(y.astype(f32), "train", -0.5, 64.0)
    pm, ps, _ = KO.lse_parts(qf, tf, items, slots, m, kind="f16")
    a = qf.view(np.float16).astype(f64) @ tf.view(np.float16).astype(f64).T
    for q0, qr, c0, c1, s, _ in items.tolist():
        lse = logsumexp(a[q0:q0 + qr, c0:c1], axis=1)
        assert np.allclose(pm[s, q0:q0 + qr] + np.log(ps[s, q0:q0 + qr]), lse, rtol=1e-14, atol=1e-12)
    # and the log-density the pair term stands for: a - |q|^2 / 2 = -|p - q|^2 / 2 up to the operands' rounding
    pm, ps, _ = KO.lse_parts(q, t, items, slots, m)
    whole = logsumexp(-0.5 * ((x[:, None, :] - y[None]) ** 2).sum(-1), axis=1)
    mine = logsumexp(pm + np.log(ps), axis=0) - 0.5 * (x * x).sum(1)
    assert np.max(np.abs(mine - whole)) <= 1e-3


def test_lse_bound_is_positive_and_grows_with_the_data():
    rng = np.random.default_rng(2)
    m, n, d = 40, 300, 8
    items, slots = E.build_items(np.array([0, m]), [[(0, n)]], 1)
    for scale in (1.0, 30.0):
        q, _ = KO.pack_lse((rng.normal(size=(m, d)) * scale).astype(f32), "query")
        t, _ = KO.pack_lse(rng.normal(size=(n, d)).astype(f32), "train")
        pm, ps, _, st = KO.lse_parts(q, t, items, slots, m, stats=True)
        bm, bl = KO.lse_bound(st, KO.k_width(d, "bf16"))
        assert np.all(bm > 0) and np.all(bl > bm)
        assert KO.lse_excess(pm, ps, pm, ps, st, KO.k_width(d, "bf16")) == (0.0, 0.0)
        # a perturbation at the bound's size is seen as such
        em, el = KO.lse_excess(pm + 2 * bm, ps, pm, ps, st, KO.k_width(d, "bf16"))
        assert em == pytest.approx(2.0) and el > 1.0


# ---- the exact construction ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["bf16", "f16"])
@pytest.mark.parametrize("d", [1, 17, 96, 97, 305])
def test_exact_construction_premise(d, kind):
    m, n = 129, 900
    q, p = KO.int_lse_operands(m, n, d, seed=d)
    assert set(np.unique(q)) <= {0.0, 8.0} and set(np.unique(p)) <= {0.0, 16.0}
    assert np.all((p != 0).sum(1) <= 1)
    d16 = -(-d // 16) * 16
    used = np.flatnonzero(np.any(p != 0, axis=0))
    assert d - 1 in used and set(used // 16) == set(range(d16 // 16))          # every K step, the last partial one too
    if kind == "bf16":
        qp, qsq = KO.pack_lse(q.astype(f32), "query")
        tp, tsq = KO.pack_lse(p.astype(f32), "train")
    else:
        qp, qsq, qflag = KO.pack_f16(q.astype(f32), "query", 0.0, KO.F16_NORM_SCALE)
        tp, tsq, tflag = KO.pack_f16(p.astype(f32), "train", -0.5, KO.F16_NORM_SCALE)
        assert not qflag and not tflag
    assert np.array_equal(qsq, (q * q).sum(1)) and np.array_equal(tsq, (p * p).sum(1))
    qv, tv = KO.decode(qp, kind), KO.decode(tp, kind)
    # every product and every partial sum of the K-loop, in K order and in any other, is an integer below 2^24
    prod = qv[:, None, :] * tv[None, :, :]
    assert np.array_equal(prod, np.round(prod))
    assert np.abs(prod).sum(-1).max() < 2 ** 24 and np.abs(np.cumsum(prod, axis=-1)).max() < 2 ** 24
    a = prod.sum(-1)
    assert set(np.unique(a)) <= {KO.HIT, KO.MISS}
    hits = np.diff(KO.hit_prefix(q, p), axis=1)
    assert np.array_equal(a == KO.HIT, hits == 1)
    # the float64 partials of the packed operands are the integer counts (up to the misses' exp(-128) terms)
    items, slots = E.build_items(np.array([0, m]), [[(0, n)]], 1)
    pm, ps, cov = KO.lse_parts(qp, tp, items, slots, m, kind=kind)
    em, es, ecov = KO.exact_lse_parts(KO.hit_prefix(q, p), items, slots)
    assert np.array_equal(cov, ecov) and np.array_equal(pm[cov], em[cov])
    assert np.allclose(ps[cov], es[cov], rtol=1e-40 + 1e-15, atol=0)
    # spans with and without a hit both occur, and zero-row columns exist
    assert np.any(em[cov] == KO.HIT) and np.any(em[cov] == KO.MISS)


def _defects(q, p, items, slots, pm, ps):
    """(name, corrupted copy of (pm, ps)) for each kernel defect, on the exact construction"""
    m, n = q.shape[0], p.shape[0]
    zero = ~np.any(p != 0, axis=1)
    k = np.argmax(p != 0, axis=1)
    hit = lambda r, j: bool(zero[j] or q[r, k[j]] != 0)
    spans = sorted({(int(c0), int(c1), int(s), int(q0), int(qr)) for q0, qr, c0, c1, s, _ in items.tolist()})
    out = []

    def with_col(name, sign, pick):
        """count one column once more (sign +1) or once less (-1) in the (slot, row) pick() names"""
        s, r, j = pick
        a, b = pm.copy(), ps.copy()
        if pm[s, r] == KO.HIT:
            if hit(r, j):
                b[s, r] += sign
                if b[s, r] == 0:                             # the only hit gone: the span has none left
                    a[s, r], b[s, r] = KO.MISS, float([c1 - c0 for c0, c1, ss, q0, qr in spans
                                                       if ss == s and q0 <= r < q0 + qr][0] - 1)
        else:
            if hit(r, j):
                a[s, r], b[s, r] = (KO.HIT, 1.0) if sign > 0 else (KO.MISS, b[s, r])
            else:
                b[s, r] += sign
        out.append((name, a, b))

    hit_entry = next((s, r, j) for c0, c1, s, q0, qr in spans for r in range(q0, q0 + qr)
                     if pm[s, r] == KO.HIT for j in range(c0, c1) if hit(r, j))
    miss_entry = next(((s, r, c0) for c0, c1, s, q0, qr in spans for r in range(q0, q0 + qr)
                       if pm[s, r] == KO.MISS), None)
    with_col("hit_column_dropped", -1, hit_entry)
    with_col("hit_column_counted_twice", +1, hit_entry)
    if miss_entry is not None:
        with_col("column_of_a_span_without_hits_dropped", -1, miss_entry)
        with_col("column_of_a_span_without_hits_counted_twice", +1, miss_entry)
    # a column past col1: the next span's first column (where it counts: a hit, or any column in a span without one)
    # or, for a span that ends at n, a zero-filled column (a = 0, a hit)
    past = next(((s, r, c1) for c0, c1, s, q0, qr in spans for r in range(q0, q0 + qr)
                 if c1 == n or hit(r, c1) or pm[s, r] == KO.MISS), None)
    s, r, j = past
    a, b = pm.copy(), ps.copy()
    if j < n and not hit(r, j):
        b[s, r] += 1                                                      # a miss in a span without hits
    elif pm[s, r] == KO.HIT:
        b[s, r] += 1
    else:
        a[s, r], b[s, r] = KO.HIT, 1.0
    out.append(("column_past_col1", a, b))
    last = [sp for sp in spans if sp[1] == n]
    c0, c1, s, q0, qr = last[0]
    a, b = pm.copy(), ps.copy()                                           # zero-filled column past n (no col1 mask)
    a[s, q0:q0 + qr] = KO.HIT
    b[s, q0:q0 + qr] = np.where(pm[s, q0:q0 + qr] == KO.HIT, ps[s, q0:q0 + qr] + 1, 1.0)
    out.append(("zero_filled_column_past_n", a, b))
    # a span written to a neighbouring slot (its own slot left unwritten)
    for c0, c1, s, q0, qr in spans:
        nb = s + 1 if s + 1 < slots else s - 1
        rows = slice(q0, q0 + qr)
        if nb >= 0 and (not np.array_equal(pm[s, rows], pm[nb, rows]) or not np.array_equal(ps[s, rows], ps[nb, rows])):
            a, b = pm.copy(), ps.copy()
            a[nb, rows], b[nb, rows] = pm[s, rows], ps[s, rows]
            a[s, rows], b[s, rows] = np.nan, np.nan
            out.append(("span_in_neighbour_slot", a, b))
            break
    a, b = pm.copy(), ps.copy()                                           # one (slot, row) entry unwritten
    s, r = hit_entry[:2]
    a[s, r], b[s, r] = np.nan, np.nan
    out.append(("entry_unwritten", a, b))
    a, b = pm.copy(), ps.copy()                                           # an entry written outside the list
    if np.any(np.isnan(pm)):
        s, r = np.argwhere(np.isnan(pm))[0]
        a[s, r], b[s, r] = KO.HIT, 1.0
        out.append(("entry_outside_the_list", a, b))
    cov = ~np.isnan(pm)                                                   # two rows swapped
    for r1 in range(m):
        for r2 in range(r1 + 1, m):
            if np.array_equal(cov[:, r1], cov[:, r2]) and not np.array_equal(ps[cov[:, r1], r1], ps[cov[:, r2], r2]):
                a, b = pm.copy(), ps.copy()
                a[:, [r1, r2]], b[:, [r1, r2]] = pm[:, [r2, r1]], ps[:, [r2, r1]]
                out.append(("rows_swapped", a, b))
                break
        else:
            continue
        break
    return out


EXACT_CASES = [(1, 100, 17, 1), (129, 129, 17, 1), (127, 700, 96, 2), (300, 2000, 97, 1), (500, 9000, 305, 16)]


@pytest.mark.parametrize("m, n, d, span_tiles", EXACT_CASES)
def test_exact_comparison_rejects_every_defect(m, n, d, span_tiles):
    q, p = KO.int_lse_operands(m, n, d, seed=m + n + d)
    items, slots = E.build_items(np.array([0, m]), [[(0, n)]], span_tiles)
    lists = {"build_items": items, "ragged": KO.ragged_items(m, n, span_tiles, seed=m)}
    applied = set()
    for name, lst in lists.items():
        slots = int(lst[:, 4].max()) + 1
        pm, ps, cov = KO.exact_lse_parts(KO.hit_prefix(q, p), lst, slots)
        assert KO.exact_excess(pm, ps, pm, ps) == 0.0
        # within the budget: 0.9 of it in either direction, in float32
        noisy = (ps * (1 + 0.9 * KO.EXACT_RTOL * np.cos(np.arange(ps.size)).reshape(ps.shape))).astype(f32)
        assert KO.exact_excess(pm.astype(f32), noisy, pm, ps) <= 1.0
        for defect, a, b in _defects(q, p, lst, slots, pm, ps):
            applied.add(defect)
            ex = KO.exact_excess(a, b, pm, ps)
            assert ex > 100.0, (name, defect, ex)
    must = {"hit_column_dropped", "hit_column_counted_twice", "column_past_col1", "zero_filled_column_past_n",
            "entry_unwritten"} | ({"rows_swapped"} if m > 1 else set())
    assert must <= applied, must - applied


def test_every_defect_applies_somewhere():
    applied = set()
    for m, n, d, span_tiles in EXACT_CASES:
        q, p = KO.int_lse_operands(m, n, d, seed=m + n + d)
        for lst in (E.build_items(np.array([0, m]), [[(0, n)]], span_tiles)[0], KO.ragged_items(m, n, span_tiles, m)):
            slots = int(lst[:, 4].max()) + 1
            pm, ps, _ = KO.exact_lse_parts(KO.hit_prefix(q, p), lst, slots)
            applied |= {name for name, _, _ in _defects(q, p, lst, slots, pm, ps)}
    assert applied == {"hit_column_dropped", "hit_column_counted_twice", "column_of_a_span_without_hits_dropped",
                       "column_of_a_span_without_hits_counted_twice", "column_past_col1", "zero_filled_column_past_n",
                       "span_in_neighbour_slot", "entry_unwritten", "entry_outside_the_list", "rows_swapped"}


# ---- work lists ------------------------------------------------------------------------------------------------
SIZES = [(m, n) for m in (1, 127, 129, 500) for n in (1, 100, 128, 129, 70_001)]


@pytest.mark.parametrize("m, n", SIZES)
def test_check_kde_work_list_accepts_the_lists_the_gpu_tests_run(m, n):
    q_off = np.array([0, m])
    pairs = E.count_tile_pairs(q_off, [[(0, n)]], 128)
    for span_tiles in sorted({1, 2, 16, E.span_tiles_for(pairs, 132), E.span_tiles_for(pairs, 114)}):
        items, slots = E.build_items(q_off, [[(0, n)]], span_tiles, 128)
        assert int(items[:, 4].max()) + 1 == slots
        for lst in (items, E.span_major(items), KO.residency_order(items, 132), KO.residency_order(items, 7)):
            KO.check_kde_work_list(lst, m, n, span_tiles)
            assert sorted(map(tuple, lst.tolist())) == sorted(map(tuple, items.tolist()))
        KO.check_kde_work_list(KO.ragged_items(m, n, span_tiles, seed=n), m, n, span_tiles)
        for g in (7, 132):
            if items.shape[0] > g and m > 128:
                assert KO.resident_pairs(KO.residency_order(items, g), g) > 0


def test_check_kde_work_list_rejects_broken_lists():
    m, n = 300, 1000
    items, _ = E.build_items(np.array([0, m]), [[(0, n)]], 1)
    KO.check_kde_work_list(items, m, n, 1)
    with pytest.raises(AssertionError):
        KO.check_kde_work_list(items, m, n, 1, col_tile=128)               # spans wider than allowed

    def broken(edit, mm=m, nn=n):
        it = items.copy()
        it = edit(it)
        with pytest.raises(AssertionError):
            KO.check_kde_work_list(it, mm, nn, 1)

    def setv(i, j, v):
        def f(it):
            it[i, j] = v(it) if callable(v) else v
            return it
        return f

    broken(setv(0, 3, lambda it: it[0, 3] - 1))                  # a column of a span dropped
    broken(setv(1, 2, lambda it: it[1, 2] - 1))                  # spans overlap
    broken(setv(-1, 1, lambda it: it[-1, 1] - 1))                # q_rows of the last tile short by one
    broken(setv(-1, 1, 128))                                     # ... or a full tile
    broken(setv(1, 4, lambda it: it[0, 4]))                      # two spans of a tile share a slot
    broken(lambda it: it[it[:, 0] != 128])                       # a query tile missing
    broken(setv(-1, 3, n + 1))                                   # col1 past n
    broken(lambda it: np.concatenate([it, it[:1]]))              # an item twice
    broken(lambda it: it, nn=n + 1)                              # the columns do not reach n


# ---- the merge of the partials ---------------------------------------------------------------------------------
def test_combine_ref_matches_logsumexp_and_handles_empty_slots():
    rng = np.random.default_rng(4)
    slots, m = 19, 50
    pm = rng.uniform(-30, 30, size=(slots, m)).astype(f32)
    ps = rng.uniform(1, 300, size=(slots, m)).astype(f32)
    pm[rng.random((slots, m)) < 0.3] = -np.inf
    pm[:, 3] = -np.inf                                        # a row without any partial
    pm[2, 7] = np.nan                                         # a NaN max is skipped like -inf
    M, S, bound = KO.combine_ref(pm, ps)
    assert M[3] == -np.inf and S[3] == 0.0 and bound[3] == 0.0
    live = pm > -np.inf
    for r in range(m):
        if r == 3:
            continue
        w = live[:, r]
        want = logsumexp(pm[w, r].astype(f64) + np.log(ps[w, r].astype(f64)))
        assert M[r] == pm[w, r].max() and abs(M[r] + math.log(S[r]) - want) <= 1e-13
    assert np.all(bound[np.arange(m) != 3] > 2.0 ** -23 * S[np.arange(m) != 3])


def test_combine_unit_replica_follows_the_slot_groups():
    """with all maxima 0 only the order of the fp32 adds is left; in groups s mod 8 it differs from ascending order"""
    slots = 17
    ps = np.ones((slots, 2), dtype=f32)
    ps[0] = 2.0 ** 24                                         # group 0 starts at 2^24: its later + 1 are lost
    pm = np.zeros((slots, 2), dtype=f32)
    pm[0, 1] = -np.inf                                        # row 1: slot 0 empty
    M, S = KO.combine_unit_replica(pm, ps)
    assert np.array_equal(M, [0.0, 0.0])
    # row 0: group 0 (slots 0, 8, 16) = 2^24, each + 1 rounds back to even; groups 1..7 (slots g, g + 8) = 2 each,
    # and 2^24 + 2 + ... + 2 = 2^24 + 14 is exact.  In ascending slot order every + 1 after the first slot is lost.
    seq = np.float32(0)
    for v in ps[:, 0]:
        seq = np.float32(seq + v)
    assert seq == 2.0 ** 24 and S[0] == 2.0 ** 24 + 14
    assert S[1] == 16.0
    empty = KO.combine_unit_replica(np.full((3, 1), -np.inf, dtype=f32), np.ones((3, 1), dtype=f32))
    assert empty[0][0] == -np.inf and empty[1][0] == 0.0


# ---- whitening reference ---------------------------------------------------------------------------------------
def test_whiten_bound_reference():
    rng = np.random.default_rng(6)
    x = rng.normal(size=(9, 12)).astype(f32)
    cols = np.array([11, 0, 5, 3], dtype=np.int32)
    mu = rng.normal(size=4)
    w = rng.normal(size=(4, 4)).astype(f32)
    ref, bound = KO.whiten_bound(x, cols, mu, w)
    assert np.allclose(ref, (x[:, cols].astype(f64) - mu) @ w.astype(f64), rtol=1e-15, atol=0)
    ref2, _ = KO.whiten_bound(x, None, mu, w)
    assert np.allclose(ref2, (x[:, :4].astype(f64) - mu) @ w.astype(f64), rtol=1e-15, atol=0)
    # fp32 products summed in fp32 in a fixed order stay inside the budget
    v = (x[:, cols].astype(f64) - mu).astype(f32)
    acc = np.zeros((9, 4), dtype=f32)
    for k in range(4):
        acc = np.float32(acc + np.float32(v[:, k:k + 1] * w[k]))
    assert np.all(np.abs(acc - ref) <= 2 * bound)     # separate mul + add: two roundings per step, twice the FMA's


# ---- host side of the density: StableGaussianKDE._finish -------------------------------------------------------
def _kde_without_device(n, norm):
    from simple_tip_b200.core.stable_kde import StableGaussianKDE

    kde = StableGaussianKDE.__new__(StableGaussianKDE)
    kde.n, kde.norm, kde.log_norm = n, norm, math.log(norm)
    return kde


@pytest.mark.parametrize("norm", [0.37, 2.0 ** -30])
def test_finish_reproduces_the_references_underflow(norm):
    """the float64 restatement of scipy 1.4.1's sum: density = sum_i fl(fl(exp(a_i) norm) w), w = 1/n.  _finish gets
    the log-domain (max a, sum exp(a - max)) exactly; its density is exactly 0 where the restatement's largest term
    is 0, and agrees to 1e-12 relative wherever the restatement's density is a normal float64 (-log density 700 ...
    760 spans the normal range, the subnormal one and exact underflow; the subnormal range is the documented
    deviation of DESIGN.md §5)"""
    rng = np.random.default_rng(3)
    n = 1000
    kde = _kde_without_device(n, norm)
    w = 1.0 / n
    rows = 3000
    target = np.linspace(700.0, 760.0, rows)                   # -log density
    k = rng.integers(1, 12, size=rows)
    log_max, rel_sum, ref, largest = (np.empty(rows) for _ in range(4))
    for i in range(rows):
        off = np.concatenate([[0.0], rng.uniform(0.0, 4.0, size=k[i] - 1)])
        s = np.sum(np.exp(-off))
        lm = -target[i] - math.log(norm) - math.log(w) - math.log(s)
        a = lm - off
        with np.errstate(under="ignore"):
            terms = (np.exp(a) * norm) * w
        log_max[i], rel_sum[i], ref[i], largest[i] = lm, s, terms.sum(), terms.max()
    got = kde._finish(log_max, rel_sum)
    assert np.all(got[largest == 0] == 0.0) and np.any(largest == 0)
    normal = ref >= np.finfo(np.float64).tiny
    assert normal.sum() > rows // 10
    rel = np.abs(got[normal] - ref[normal]) / ref[normal]
    assert rel.max() <= 1e-12, rel.max()
    # the log-domain inputs a non-finite max stands for: no partial at all
    assert np.array_equal(kde._finish(np.array([-np.inf]), np.array([0.0])), [0.0])
