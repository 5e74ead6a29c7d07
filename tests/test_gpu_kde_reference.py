"""GPU tests of the LSA kernels against float64 references of their own operands (oracle/kde_oracle.py), through the C
ABI:

  * the packing of tip_pair_prep (LSA's arguments) and tip_pair_prep_f16 bit for bit, sqnorm to 1 fp32 ulp, and the
    fp16 range flag exactly where the emulation raises it;
  * tip_kde_lse and tip_kde_lse_f16 on the exact construction: part_max exactly 0 or -128 and part_sum the integer
    hit count (or the span width) within 2^-20 of it, every covered (slot, row) written and nothing else (the outputs
    are NaN-filled first), for the resident-query and the streaming kernel, 1-, 2- and 16-tile spans and the card's
    own choice, in build_items order, span-major order, an order in which each CTA runs consecutive items on one
    query tile (the kernel then keeps the tile in shared memory), and spans of random widths;
  * both passes on real-valued operands within lse_bound, tip_kde_combine within combine_ref's bound (and bit for bit
    where only the order of its fp32 adds is left), KdeEngine.log_kernel_sum end to end on the exact construction;
  * tip_whiten and tip_row_sqnorm bit for bit on integer data and within whiten_bound on real data;
  * the fit-time fp16 range check of KdeEngine.
Lines starting with [kde-ref] report the worst errors (run with -s to see them)."""
import math
import time

import numpy as np
import pytest

from oracle import kde_oracle as KO
from oracle import sil_oracle as SO

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64
NAN_BF16, NAN_F16 = 0x7FC1, 0x7E01          # NaN bit patterns the outputs start as


def _env():
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    return torch, _lib, _lib.load(), E


def _dev(a):
    torch = _env()[0]
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _packed(bits, kind):
    """uint16 bit patterns -> a device bf16 / fp16 matrix"""
    torch = _env()[0]
    return _dev(np.asarray(bits, dtype=np.uint16).view(np.int16)).view(torch.bfloat16 if kind == "bf16" else torch.float16)


def _bits(t):
    return t.view(_env()[0].int16).cpu().numpy().view(np.uint16)


def _sms():
    _, _, lib, E = _env()
    return E._device_sms(lib)


# ---- packing ---------------------------------------------------------------------------------------------------
def _prep3(xd, cen, role):
    torch, _lib, lib, E = _env()
    n, d = xd.shape
    out = torch.full((n, int(lib.tip_pair_pitch(d, 3))), NAN_BF16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    sq = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(lib.tip_pair_prep(E._p(xd), E.tip_dtype(xd.dtype), n, d, E._p(cen), _lib.ROLE_TRAIN if role == "train"
                                 else _lib.ROLE_QUERY, 3, 1.0, -0.5 if role == "train" else 0.0, E._p(out), E._p(sq),
                                 None, E._stream()), "tip_pair_prep")
    return _bits(out), sq.cpu().numpy()


def _prep16(xd, cen, role, S=KO.F16_NORM_SCALE):
    torch, _lib, lib, E = _env()
    n, d = xd.shape
    out = torch.full((n, int(lib.tip_pair_pitch(d, 1))), NAN_F16, dtype=torch.int16, device="cuda").view(torch.float16)
    sq = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(lib.tip_pair_prep_f16(E._p(xd), E.tip_dtype(xd.dtype), n, d, E._p(cen), _lib.ROLE_TRAIN if role == "train"
                                     else _lib.ROLE_QUERY, -0.5 if role == "train" else 0.0, S, E._p(out), E._p(sq),
                                     E._p(flags), E._stream()), "tip_pair_prep_f16")
    return _bits(out), sq.cpu().numpy(), bool(flags.item())


@pytest.mark.parametrize("dtype", [f32, f64])
@pytest.mark.parametrize("d", [1, 15, 16, 17, 96, 97, 256, 304, 305, 2048])
def test_lse_packing_is_bit_for_bit(d, dtype):
    rng = np.random.default_rng(d * 2 + (dtype == f64))
    n = 300
    x = (rng.normal(size=(n, d)) * np.exp(rng.normal(size=(n, 1)) * 2.0)).astype(dtype)
    center = (rng.normal(size=d) * 0.5).astype(f32)
    x[5], x[6], x[7] = 0.0, -0.0, center                 # zero rows and a row on the centre (v = 0)
    x[8] = np.round(x[8] * 8) / 8                         # bf16-exact values: l = 0
    x[9] = rng.integers(-8, 9, size=d)                    # the exact construction's kind of row
    xd = _dev(x)
    d16 = -(-d // 16) * 16
    tail3 = np.zeros(SO.pair_pitch(d), dtype=bool)
    tail3[3 * d16:3 * d16 + 3] = True
    tail1 = np.zeros(KO.pair_pitch1(d), dtype=bool)
    tail1[d16:d16 + 3] = True
    ulp = lambda a, b: np.all(np.abs(a.astype(f64) - b) <= np.spacing(np.abs(b)))
    for cen in (None, center):
        cd = None if cen is None else _dev(cen)
        for role in ("query", "train"):
            where = f"d={d} {np.dtype(dtype).name} center={cen is not None} {role}"
            got, gsq = _prep3(xd, cd, role)
            want, wsq = KO.pack_lse(x, role, cen)
            assert np.array_equal(got[:, ~tail3], want[:, ~tail3]), (where, np.argwhere(got[:, ~tail3] != want[:, ~tail3])[:4].tolist())
            assert ulp(gsq, wsq), where
            # the train tail is the split of the norm the kernel reports; the query tail is 1, 1, 1
            tail = SO.bf16_bits(KO.lse_tail(gsq)) if role == "train" else want[:, tail3]
            assert np.array_equal(got[:, tail3], tail), where
            got, gsq, gflag = _prep16(xd, cd, role)
            want, wsq, wflag = KO.pack_f16(x, role, -0.5 if role == "train" else 0.0, KO.F16_NORM_SCALE, cen)
            assert np.array_equal(got[:, ~tail1], want[:, ~tail1]), (where, np.argwhere(got[:, ~tail1] != want[:, ~tail1])[:4].tolist())
            assert ulp(gsq, wsq), where
            # the train tail from the kernel's norm; a norm term past fp16's range gives inf and then NaN, whose
            # payload is not specified
            tail = KO.f16_tail(gsq, -0.5, KO.F16_NORM_SCALE)[0].view(np.uint16) if role == "train" else want[:, tail1]
            nan = np.isnan(KO.decode(tail, "f16"))
            assert np.array_equal(np.isnan(KO.decode(got[:, tail1], "f16")), nan), where
            assert np.array_equal(got[:, tail1][~nan], tail[~nan]), where
            assert gflag == wflag, where


FLAG_CASES = [("max_finite", [[65504.0, -65504.0]], "query", False), ("rounds_to_inf", [[1.0, 65520.0]], "query", True),
              ("inf", [[1.0, np.inf]], "query", True), ("nan", [[np.nan, 1.0]], "query", True),
              ("nan_train", [[np.nan, 1.0]], "train", True), ("norm_past_range", [[2896.0, 0.0]], "train", True),
              ("norm_inside_range", [[2895.0, 0.0]], "train", False), ("norm_of_a_query", [[2896.0, 0.0]], "query", False),
              ("max_finite_train", [[65504.0, 0.0]], "train", True)]


@pytest.mark.parametrize("name, rows, role, want", FLAG_CASES, ids=[c[0] for c in FLAG_CASES])
def test_f16_flag_is_raised_exactly_where_the_emulation_raises_it(name, rows, role, want):
    rng = np.random.default_rng(1)
    for dtype in (f32, f64):
        # the row sits at position 203 of 300 ordinary rows (another block and warp than the first)
        x = rng.normal(size=(300, 2))
        x[203] = rows[0]
        x = x.astype(dtype)
        assert KO.pack_f16(x, role, -0.5 if role == "train" else 0.0, KO.F16_NORM_SCALE)[2] == want
        assert _prep16(_dev(x), None, role)[2] == want, (name, np.dtype(dtype).name)
        x[203] = 0.5
        assert not _prep16(_dev(x), None, role)[2]


# ---- exact partials --------------------------------------------------------------------------------------------
def _operands(kind, q, p):
    """device packs of the exact construction, from the emulation (the packing test above checks the kernels)"""
    if kind == "bf16":
        qb, _ = KO.pack_lse(q.astype(f32), "query")
        tb, _ = KO.pack_lse(p.astype(f32), "train")
    else:
        qb, _, qf = KO.pack_f16(q.astype(f32), "query", 0.0, KO.F16_NORM_SCALE)
        tb, _, tf = KO.pack_f16(p.astype(f32), "train", -0.5, KO.F16_NORM_SCALE)
        assert not qf and not tf
    return qb, tb, _packed(qb, kind), _packed(tb, kind)


def _lse(kind, qd, m, td, n, d, items, slots):
    """one tip_kde_lse / tip_kde_lse_f16 launch into NaN-filled partials"""
    torch, _lib, lib, E = _env()
    pm = torch.full((slots, m), float("nan"), dtype=torch.float32, device="cuda")
    ps = torch.full((slots, m), float("nan"), dtype=torch.float32, device="cuda")
    it = _dev(np.ascontiguousarray(items, dtype=np.int32))
    fn, segs = (lib.tip_kde_lse, 3) if kind == "bf16" else (lib.tip_kde_lse_f16, 1)
    _lib.check(fn(E._p(qd), m, E._p(td), n, d, int(lib.tip_pair_pitch(d, segs)), E._p(it), items.shape[0], E._p(pm),
                  E._p(ps), E._stream()), "tip_kde_lse" + ("_f16" if kind == "f16" else ""))
    return pm.cpu().numpy(), ps.cpu().numpy()


def _resident(kind, d):
    """the kernel tip_kde_lse* runs: resident query tile while the packed row fits 5 K chunks of 64"""
    return (KO.k_width(d, kind) // 16 + 3) // 4 <= 5


@pytest.mark.parametrize("d", [17, 96, 97, 300])
def test_integer_operands_accumulate_exactly(d):
    """the premise of the exact case: on these operands the K-loop yields a = 0 or -128 exactly, in the
    resident-query kernel (d <= 96) and in the streaming one"""
    torch, _lib, lib, E = _env()
    q, p = KO.int_lse_operands(128, 256, d, seed=d)
    _, _, qd, td = _operands("bf16", q, p)
    want = np.where(np.diff(KO.hit_prefix(q, p), axis=1) == 1, KO.HIT, KO.MISS)
    for variant in ((1, 2) if d <= 96 else (1,)):
        out = torch.full((256, 256), float("nan"), dtype=torch.float32, device="cuda")
        _lib.check(lib.tip_pair_probe(E._p(qd), 128, E._p(td), 256, d, 3, int(lib.tip_pair_pitch(d, 3)), variant,
                                      E._p(out), E._stream()), "tip_pair_probe")
        got = out[:128].cpu().numpy().astype(f64)
        assert np.array_equal(got, want), (d, variant, float(np.nanmax(np.abs(got - want))))


EXACT = [("bf16", 17), ("bf16", 96), ("bf16", 97), ("bf16", 300), ("f16", 17), ("f16", 304), ("f16", 305)]
SIZES = [(m, n) for n in (1, 100, 128, 129, 70_001) for m in (1, 127, 129, 500)]


@pytest.mark.parametrize("kind, d", EXACT, ids=[f"{k}-d{d}" for k, d in EXACT])
def test_kde_lse_exact_partials(kind, d):
    torch, _lib, lib, E = _env()
    assert int(lib.tip_kde_slot_parts()) == 1 and int(lib.tip_kde_tile_rows()) == KO.ROW_TILE
    sms = _sms()
    t0 = time.time()
    worst, worst_abs, ex2_err, launches, resident_runs, unwritten = 0.0, 0.0, 0.0, 0, 0, 0
    for m, n in SIZES:
        q, p = KO.int_lse_operands(m, n, d, seed=m * 7 + n + d)
        _, _, qd, td = _operands(kind, q, p)
        prefix = KO.hit_prefix(q, p)
        q_off = np.array([0, m])
        pairs = E.count_tile_pairs(q_off, [[(0, n)]], KO.ROW_TILE)
        for span_tiles in sorted({1, 2, 16, E.span_tiles_for(pairs, sms)}):
            items, _ = E.build_items(q_off, [[(0, n)]], span_tiles, KO.ROW_TILE)
            g = min(items.shape[0], sms)              # the kernel's persistent grid
            lists = {"build_items": items, "span_major": E.span_major(items),
                     "resident": KO.residency_order(items, g),
                     "ragged": KO.ragged_items(m, n, span_tiles, seed=m + n + span_tiles)}
            for name, lst in lists.items():
                KO.check_kde_work_list(lst, m, n, span_tiles)
                slots = int(lst[:, 4].max()) + 1
                pm, ps = _lse(kind, qd, m, td, n, d, lst, slots)
                launches += 1
                rm, rs, cov = KO.exact_lse_parts(prefix, lst, slots)
                unwritten += int(np.sum(cov & np.isnan(pm)))
                ex = KO.exact_excess(pm, ps, rm, rs)
                where = (kind, d, m, n, span_tiles, name)
                if not np.isfinite(ex):
                    bad = np.argwhere(cov & ~((pm == rm) & np.isfinite(ps)) | (~cov & ~np.isnan(pm)))[:4]
                    raise AssertionError((where, "entries", bad.tolist(), [(pm[s, r], ps[s, r], rm[s, r], rs[s, r])
                                                                          for s, r in bad]))
                assert ex <= 1.0, (where, ex)
                worst = max(worst, ex)
                worst_abs = max(worst_abs, float(np.max(np.abs(ps[cov] - rs[cov]), initial=0.0)))
                miss = cov & (rm == KO.MISS)
                if miss.any():
                    ex2_err = max(ex2_err, float(np.max(np.abs(ps[miss] / rs[miss] - 1.0))))
                if name == "resident":
                    resident_runs += KO.resident_pairs(lst, g)
    # the residency path: some CTA ran items w and w + G on one query tile (m = 500 against 70 001 columns has more
    # items than any H100 has SMs)
    assert resident_runs > 0
    print(f"[kde-ref] exact partials {kind} d={d} ({'resident' if _resident(kind, d) else 'streaming'} kernel, "
          f"{sms} SMs): {launches} launches, worst |part_sum - count| {worst_abs:.3g} = {worst:.3g} of 2^-20 count, "
          f"relative error of spans without a hit (ex2.approx(0) terms) {ex2_err:.3g}, unwritten entries {unwritten}, "
          f"consecutive items on a resident query tile {resident_runs}, {time.time() - t0:.1f} s")


# ---- real-valued partials --------------------------------------------------------------------------------------
def _real_case(m, n, d, seed):
    """whitened Gaussian clusters (as StableGaussianKDE whitens them: Scott factor, Cholesky of the inverse
    covariance); columns sorted along one direction so that queries out there meet a rising maximum (a rescale in
    most chunks); queries from the data, from a far cluster along that direction, and scaled up to |a| ~ 10^3"""
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(5, d)) * 2.0
    raw = centres[rng.integers(0, 5, size=n)] + rng.normal(size=(n, d)) * 0.7
    mean = raw.mean(0)
    factor = n ** (-1.0 / (d + 4))
    w = np.linalg.cholesky(np.linalg.inv(np.cov(raw.T) * factor ** 2))
    p = (raw - mean) @ w
    u = rng.normal(size=d)
    u /= np.linalg.norm(u)
    p = p[np.argsort(p @ u)]
    q = ((centres[rng.integers(0, 5, size=m)] + rng.normal(size=(m, d)) * 0.7) - mean) @ w
    far = np.arange(m) % 5 == 1
    q[far] += 2.0 * np.abs(p @ u).max() * u
    big = np.arange(m) % 5 == 3
    q[big] *= 1000.0 / max(1.0, float(np.median(np.abs(q[big] @ p[::max(1, n // 500)].T))))
    return q, p


REAL = [("bf16", 32), ("bf16", 200), ("f16", 64), ("f16", 400)]


@pytest.mark.parametrize("kind, d", REAL, ids=[f"{k}-d{d}" for k, d in REAL])
def test_kde_lse_real_partials_within_bound(kind, d):
    _, _, lib, E = _env()
    m, n = 300, 20_000
    q, p = _real_case(m, n, d, seed=d)
    qb, tb, qd, td = _operands(kind, q, p) if kind == "bf16" else _f16_operands(q, p)
    amax = 0.0
    out = []
    for span_tiles in (2, 16):
        items, _ = E.build_items(np.array([0, m]), [[(0, n)]], span_tiles, KO.ROW_TILE)
        lst = KO.residency_order(items, min(items.shape[0], _sms()))
        slots = int(lst[:, 4].max()) + 1
        pm, ps = _lse(kind, qd, m, td, n, d, lst, slots)
        rm, rs, cov, st = KO.lse_parts(qb, tb, lst, slots, m, kind=kind, device="cuda", stats=True)
        em, el = KO.lse_excess(pm, ps, rm, rs, st, KO.k_width(d, kind))
        amax = max(amax, float(np.nanmax(st["amax"])))
        err = np.abs((pm + np.log(ps))[cov] - (rm + np.log(rs))[cov])
        out.append((span_tiles, em, el, float(err.max())))
        assert em <= 1.0 and el <= 1.0, (kind, d, span_tiles, em, el)
    print(f"[kde-ref] real partials {kind} d={d} (max |a| {amax:.3g}): worst err / bound of part_max and of "
          f"part_max + log part_sum per span width: "
          + ", ".join(f"{s} tiles {em:.3g} / {el:.3g} (|err| {e:.3g})" for s, em, el, e in out))


def _f16_operands(q, p):
    qb, _, qf = KO.pack_f16(q.astype(f32), "query", 0.0, KO.F16_NORM_SCALE)
    tb, _, tf = KO.pack_f16(p.astype(f32), "train", -0.5, KO.F16_NORM_SCALE)
    assert not qf and not tf
    return qb, tb, _packed(qb, "f16"), _packed(tb, "f16")


# ---- the merge of the partials ---------------------------------------------------------------------------------
def _combine(pm, ps):
    torch, _lib, lib, E = _env()
    slots, m = pm.shape
    om = torch.full((m,), float("nan"), dtype=torch.float32, device="cuda")
    os_ = torch.full((m,), float("nan"), dtype=torch.float32, device="cuda")
    pmd, psd = _dev(pm), _dev(ps)          # held until the launch has read them
    _lib.check(lib.tip_kde_combine(E._p(pmd), E._p(psd), m, slots, E._p(om), E._p(os_), E._stream()), "tip_kde_combine")
    return om.cpu().numpy(), os_.cpu().numpy()


@pytest.mark.parametrize("slots", [1, 7, 8, 9, 64, 300])
def test_kde_combine_within_bound(slots):
    rng = np.random.default_rng(slots)
    worst = {}
    for m in (1, 31, 32, 33, 100_003):
        for case in ("random", "empty_slots", "apart_100"):
            pm = rng.uniform(-50.0, 50.0, size=(slots, m)).astype(f32)
            ps = rng.uniform(1.0, 4096.0, size=(slots, m)).astype(f32)
            if case == "empty_slots":
                empty = rng.random((slots, m)) < 0.5
                pm[empty], ps[empty] = -np.inf, 0.0
                pm[:, ::7], ps[:, ::7] = -np.inf, 0.0            # rows with every slot empty
            elif case == "apart_100":
                pm = np.where(rng.random((slots, m)) < 0.5, 0.0, -100.0).astype(f32)
            om, os_ = _combine(pm, ps)
            ratio = 0.0
            for r0 in range(0, m, 20_000):
                sl = slice(r0, min(m, r0 + 20_000))
                M, S, bound = KO.combine_ref(pm[:, sl], ps[:, sl])
                empty_row = ~np.isfinite(M)
                assert np.array_equal(om[sl], M.astype(f32)), (slots, m, case)
                assert np.all(os_[sl][empty_row] == 0.0), (slots, m, case)
                err = np.abs(os_[sl].astype(f64) - S)
                assert np.all(err <= bound), (slots, m, case, float(np.max(err[~empty_row] / bound[~empty_row])))
                if (~empty_row).any():
                    ratio = max(ratio, float(np.max(err[~empty_row] / bound[~empty_row])))
            worst[(m, case)] = ratio
    print(f"[kde-ref] combine slots={slots}: worst |err| / bound {max(worst.values()):.3g} "
          f"(random {max(v for (mm, c), v in worst.items() if c == 'random'):.3g}, "
          f"maxima 100 apart {max(v for (mm, c), v in worst.items() if c == 'apart_100'):.3g})")


@pytest.mark.parametrize("slots", [1, 8, 9, 17, 300])
def test_kde_combine_is_exact_on_unit_partials(slots):
    """maxima 0 or -inf and integer sums: every factor is expf(0) = 1, and the result is the kernel's fp32 adds in its
    documented order (groups of slots s mod 8), bit for bit; 2^24 partials make that order visible"""
    rng = np.random.default_rng(slots + 1)
    m = 1000
    pm = np.where(rng.random((slots, m)) < 0.8, 0.0, -np.inf).astype(f32)
    pm[:, 5] = -np.inf
    ps = rng.integers(0, 4097, size=(slots, m)).astype(f32)
    ps[0, ::3] = 2.0 ** 24
    om, os_ = _combine(pm, ps)
    M, S = KO.combine_unit_replica(pm, ps)
    assert np.array_equal(om, M) and om[5] == -np.inf and os_[5] == 0.0
    assert np.array_equal(os_.view(np.uint32), S.view(np.uint32)), np.argwhere(os_ != S)[:4].tolist()
    small = ps < 2.0 ** 24
    exact = np.where((pm == 0) & small, ps.astype(f64), 0.0).sum(0)
    only_small = np.all(small | (pm != 0), axis=0)
    assert np.array_equal(os_[only_small].astype(f64), exact[only_small])   # integer sums below 2^24 are exact
    print(f"[kde-ref] combine slots={slots} on (0, integer) partials: bit-exact")


# ---- the engine end to end on the exact construction -----------------------------------------------------------
@pytest.mark.parametrize("m, n, d", [(129, 1000, 17), (500, 70_001, 97), (1030, 3000, 304)])
def test_engine_log_kernel_sum_exact(m, n, d):
    torch, _, _, E = _env()
    q, p = KO.int_lse_operands(m, n, d, seed=n + d)
    eng = E.KdeEngine(p)
    assert eng.fast_ok and eng.t_pack_f16 is not None
    hits = KO.hit_prefix(q, p)[:, n].astype(f64)
    want_mx = np.where(hits > 0, KO.HIT, KO.MISS)
    want_sm = np.where(hits > 0, hits, float(n))
    qd = _dev(q.astype(f32))
    for fast in (False, True):
        mx, sm, qsq = (t.cpu().numpy() for t in eng.log_kernel_sum(qd, fast=fast))
        assert np.array_equal(qsq, (q * q).sum(1).astype(f32)), fast
        assert np.array_equal(mx, want_mx), (fast, np.argwhere(mx != want_mx)[:4].tolist())
        err = np.abs(sm - want_sm) / (KO.EXACT_RTOL * want_sm)
        assert err.max() <= 1.0, (fast, float(err.max()), np.argwhere(err > 1)[:4].tolist())
        if fast:
            assert int(eng.flags.item()) == 0
        print(f"[kde-ref] engine m={m} n={n} d={d} fast={fast}: slots {eng._work_items(m)[2]}, worst |sm - count| "
              f"{float(np.max(np.abs(sm - want_sm))):.3g}")


def test_fit_time_f16_range_check():
    """a training row whose norm term -|p|^2 / 2 / 64 just leaves fp16's range retires the fast operand at fit time;
    just inside it does not (|p|^2 = 2896^2 = 8 386 816 > 64 * 2 * 65504 >= 2895^2)"""
    _, _, _, E = _env()
    rng = np.random.default_rng(9)
    p = rng.normal(size=(300, 4)) * 0.5
    for value, ok in ((2896.0, False), (2895.0, True)):
        p[17] = [value, 0.0, 0.0, 0.0]
        eng = E.KdeEngine(p)
        assert eng.fast_ok is ok, value
        assert (eng.t_pack_f16 is None) == (not ok), value


# ---- whitening -------------------------------------------------------------------------------------------------
def _whiten(x, cols, mu, w):
    torch, _lib, lib, E = _env()
    m, d_in = x.shape
    dn = w.shape[0]
    out = torch.full((m, dn), float("nan"), dtype=torch.float32, device="cuda")
    xd, cd, mud, wd = _dev(x), None if cols is None else _dev(cols), _dev(mu), _dev(w)
    _lib.check(lib.tip_whiten(E._p(xd), E.tip_dtype(x.dtype), m, d_in, E._p(cd), dn, E._p(mud), E._p(wd), E._p(out),
                              E._stream()), "tip_whiten")
    sq = torch.full((m,), float("nan"), dtype=torch.float64, device="cuda")
    _lib.check(lib.tip_row_sqnorm(E._p(out), m, dn, E._p(sq), E._stream()), "tip_row_sqnorm")
    return out.cpu().numpy(), sq.cpu().numpy()


def _whiten_inputs(m, dn, layout, dtype, integer, rng):
    d_in = dn if layout == "plain" else dn + 7
    if integer:
        x = rng.integers(-4, 5, size=(m, d_in)).astype(dtype)
        mu = rng.integers(-2, 3, size=dn).astype(f64)
        w = rng.integers(-2, 3, size=(dn, dn)).astype(f32)
    else:
        x = (rng.normal(size=(m, d_in)) * 3.0 + 1.0).astype(dtype)
        mu = rng.normal(size=dn) + 1.0
        w = (rng.normal(size=(dn, dn)) / math.sqrt(dn)).astype(f32)
    cols = rng.permutation(d_in)[:dn].astype(np.int32) if layout == "cols" else None
    return x, cols, mu, w


@pytest.mark.parametrize("dn", [1, 3, 4, 63, 64, 65, 130, 2304])
def test_whiten_and_row_sqnorm(dn):
    rng = np.random.default_rng(dn)
    worst_w, worst_s = 0.0, 0.0
    for m in (1, 127, 128, 129):
        for layout, dtype in (("plain", f32), ("cols", f64), ("cols", f32), ("wide", f64)):
            # integer data: every partial sum of the FMA chain is an integer below 2^24, so the output is exact
            x, cols, mu, w = _whiten_inputs(m, dn, layout, dtype, True, rng)
            y, sq = _whiten(x, cols, mu, w)
            ref, _ = KO.whiten_bound(x, cols, mu, w)
            assert np.abs(ref).max() < 2 ** 24 and np.array_equal(y.astype(f64), ref), (dn, m, layout)
            assert np.array_equal(sq, (ref * ref).sum(1)), (dn, m, layout)
            # real data: within the FMA chain's budget; the double row norm to (dn + 2) 2^-53 of itself
            x, cols, mu, w = _whiten_inputs(m, dn, layout, dtype, False, rng)
            y, sq = _whiten(x, cols, mu, w)
            ref, bound = KO.whiten_bound(x, cols, mu, w)
            r = np.abs(y.astype(f64) - ref) / bound
            assert r.max() <= 1.0, (dn, m, layout, float(r.max()))
            worst_w = max(worst_w, float(r.max()))
            y64 = y.astype(f64)
            want = (y64 * y64).sum(1)
            rs = np.abs(sq - want) / ((dn + 2) * 2.0 ** -53 * want + 1e-300)
            assert rs.max() <= 1.0, (dn, m, layout, float(rs.max()))
            worst_s = max(worst_s, float(rs.max()))
    print(f"[kde-ref] whiten d_out={dn}: integer data bit-exact; real data worst |err| / bound {worst_w:.3g}, "
          f"row_sqnorm {worst_s:.3g} of (d + 2) 2^-53")
