"""GPU tests of the exact re-rank (csrc/rerank.cu) and of the kernels that hand its winners on (the fused next-stage
query pack and seeds, the fused result scatter, tip_dsa_pack_out, tip_gather_rows, tip_shard_winner_queries and the
tip_comm_* exchange at world 1), through the C ABI, bit for bit against oracle/rerank_oracle.py:

  * every trace width from 1 to 136 and the leaf-program / generic-routine widths up to 2^23 + 1, through the list
    kernel and the exhaustive scan, in both modes, with exact zeros and +-0 coordinates, differences whose squares
    are subnormal, squares that overflow (every candidate at +inf: inf and the lowest gid) and +inf rows mixed with
    finite ones;
  * the list contract (negative starts, bits past n, rows of the wrong range, duplicates, empty masks, cnt == cap
    against cap + 1 and 0, cap in {1, 3, 4, 64}, ties over the four 8-lane groups, t_gid NULL);
  * the scan at queue lengths around both edges of its slicing, empty / one-row classes, n = 0, q_class NULL, the
    queue re-armed after every call and a work buffer reused; count_overflow_only; q_idx;
  * argument checks that return before any launch.
Every output starts as 0xAB bytes and is followed by a guard region (the work buffer included), so an entry never
written, or a write past a buffer, shows up."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import np_oracle
from oracle import rerank_oracle as RO

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64
GUARD = 256
FILL = 0xAB
INF32 = 0x7F800000


def _env():
    import torch

    from simple_tip_b200 import _lib

    return torch, _lib, _lib.load()


def _tip(dt):
    return 0 if dt == f32 else 1


def _dev(a):
    torch = _env()[0]
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    return _env()[0].cuda.current_stream().cuda_stream


class Buf:
    """`nbytes` of device memory followed by a guard region; every byte 0xAB, or the payload zero-filled."""

    def __init__(self, nbytes, zero=False):
        torch = _env()[0]
        self.n = int(nbytes)
        self.t = torch.full((self.n + GUARD,), FILL, dtype=torch.uint8, device="cuda")
        if zero:
            self.t[:self.n].zero_()

    @property
    def ptr(self):
        return self.t.data_ptr()

    def get(self, dtype, shape=None):
        a = self.t[:self.n].cpu().numpy().view(dtype)
        return a if shape is None else a.reshape(shape)

    def guard_ok(self):
        return bool((self.t[self.n:] == FILL).all().item())


def _same(a, b):
    """bit-identical, except that any NaN equals any NaN"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        u = np.uint32 if a.dtype == f32 else np.uint64
        nan = np.isnan(a) & np.isnan(b)
        return a.shape == b.shape and bool(np.all(nan | (a.view(u) == b.view(u))))
    return np.array_equal(a, b)


def _ptr(keep, a, dtype=None):
    if a is None:
        return None
    t = _dev(np.asarray(a, dtype=dtype))
    keep.append(t)
    return t.data_ptr()


def rerank(dt, q, t, class_off, q_class, mode, cand=None, cap=1, t_gid=None, q_idx=None, nxt=None, fin=None,
           count_only=False, work=None, stats0=(5, 7), rows=True):
    """One tip_nn_rerank call; returns its outputs as NumPy arrays (r["work"] is the work buffer, for reuse)."""
    torch, _lib, lib = _env()
    q = np.ascontiguousarray(q, dtype=dt)
    t = np.ascontiguousarray(t, dtype=dt)
    n, d = t.shape[0], q.shape[1]
    m = q.shape[0] if q_idx is None else len(q_idx)
    es = np.dtype(dt).itemsize
    keep = []
    t_ptr = _ptr(keep, t if n else np.zeros((1, d), dt))
    o = {"dist": Buf(m * es), "pos": Buf(m * 4), "gid": Buf(m * 4)}
    if rows:
        o["rows"] = Buf(m * d * es)
    wb = lib.tip_nn_rerank_work_bytes(m, _tip(dt))
    work = work if work is not None else Buf(wb, zero=True)
    assert work.n == wb
    stats = _dev(np.array(stats0, dtype=np.int64))
    ex = _lib.RerankExtras()
    ex.q_idx = _ptr(keep, q_idx, np.int32)
    ex.count_overflow_only = 1 if count_only else 0
    nx = {}
    pitch = lib.tip_pair_pitch(d, 1)
    if nxt is not None:
        nx = {"pack": Buf(m * pitch * 2), "sqnorm": Buf(m * 4), "row_min": Buf(m * 4), "cand_cnt": Buf(m * 4)}
        if nxt.get("rounderr", True):
            nx["rounderr"] = Buf(m * 4)
        if nxt.get("seed") is not None:
            ub, ex.next_t_rmax, ex.next_t_errmax = nxt["seed"]
            ex.next_seed_ub = _ptr(keep, ub, np.float32)
    if fin is not None:
        ex.fin_dist_a = _ptr(keep, fin["dist_a"], dt)
        ex.fin_gid = _ptr(keep, fin["gid"], np.int32)
        ex.fin_idx = _ptr(keep, fin.get("idx"), np.int32)
        ex.fin_n_total = fin["n_total"]
        o["fin"] = Buf(4 * fin["n_total"] * 8)
        ex.fin_out = o["fin"].ptr
    cand_idx, cand_cnt = cand if cand is not None else (None, None)
    torch.cuda.synchronize()
    rc = lib.tip_nn_rerank(_ptr(keep, q), t_ptr, _tip(dt), m, n, d, _ptr(keep, cand_idx, np.int32),
                           _ptr(keep, cand_cnt, np.int32), cap, _ptr(keep, q_class, np.int32),
                           _ptr(keep, class_off, np.int32), len(class_off) - 1, mode, _ptr(keep, t_gid, np.int32),
                           o["dist"].ptr, o["pos"].ptr, o["gid"].ptr, o["rows"].ptr if rows else None, work.ptr,
                           stats.data_ptr(), _ptr(keep, (nxt or {}).get("center"), np.float32),
                           nx["pack"].ptr if nx else None, nx["sqnorm"].ptr if nx else None,
                           nx["rounderr"].ptr if "rounderr" in nx else None, nx["row_min"].ptr if nx else None,
                           nx["cand_cnt"].ptr if nx else None, C.byref(ex), _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.tip_last_error()
    for b in list(o.values()) + list(nx.values()) + [work]:
        assert b.guard_ok(), "write past the end of a buffer"
    r = {"dist": o["dist"].get(dt), "pos": o["pos"].get(np.int32), "gid": o["gid"].get(np.int32),
         "stats": stats.cpu().numpy() - np.array(stats0), "work": work, "wordsw": work.get(np.int32)[:m + 2]}
    if rows:
        r["rows"] = o["rows"].get(dt, (m, d))
    if fin is not None:
        r["fin"] = o["fin"].get(np.float64, (4, fin["n_total"]))
    for k, b in nx.items():
        r["next_" + k] = b.get(np.uint16 if k == "pack" else np.uint32, (m, pitch) if k == "pack" else None)
    if not count_only:
        assert r["wordsw"][0] == 0 and r["wordsw"][1 + m] == 0, "queue / completion counter not re-armed"
    return r


def check(r, want, rows=True):
    assert _same(r["dist"], want["out_dist"])
    assert np.array_equal(r["pos"], want["out_pos"])
    assert np.array_equal(r["gid"], want["out_gid"])
    if rows:
        assert _same(r["rows"], want["out_rows"])
    assert r["stats"][0] == want["scanned"] and r["stats"][1] == 0


# ---- widths x values -----------------------------------------------------------------------------------------------
def _huge(dt):
    return 3e19 if dt == f32 else 1e200      # |x - y| ~ 2 of these: the square overflows


def _tiny(dt):
    return 1e-20 if dt == f32 else 1e-160    # squares below the smallest normal


def _width_case(dt, d, seed):
    rng = np.random.default_rng(seed)
    per = 3 if d > 4096 else 8
    n = 3 * per
    H, e = _huge(dt), _tiny(dt)
    t = (rng.normal(size=(n, d)) * 2 + rng.normal(size=(1, d))).astype(dt)
    t[0] = np.copysign(np.zeros(d), rng.normal(size=d))                     # +-0 coordinates
    t[1] = e * rng.normal(size=d)
    t[per:2 * per] = H * (1 + rng.random((per, d)) * 1e-3)                  # class 1: far out
    t[per + 1] = t[per]                                                     # tied at +inf
    t[2 * per:2 * per + per // 2] = H * (1 + rng.random((per // 2, d)))     # class 2: half far out, half finite
    q = (rng.normal(size=(6, d)) * 2).astype(dt)
    q[1] = -t[0]                                                            # distance exactly 0, signs flipped
    q[2] = e * rng.normal(size=d)                                           # subnormal squares against rows 0 and 1
    q[3] = -H
    q[5] = -H
    q_class = np.array([0, 0, 0, 1, 2, 2], dtype=np.int32)
    class_off = np.array([0, per, 2 * per, n], dtype=np.int32)
    gid = (n - 1 - np.arange(n)).astype(np.int32)                           # reverses position order
    cap = 4
    idx = np.zeros((6, cap, 2), dtype=np.int32)
    idx[:, 0] = (0, -1)                                                     # every row (n <= 32)
    idx[:, 1:, 0] = rng.integers(-31, n, size=(6, cap - 1))
    idx[:, 1:, 1] = rng.integers(0, 1 << 32, size=(6, cap - 1), dtype=np.int64).astype(np.uint32).view(np.int32)
    cnt = rng.integers(1, cap + 1, size=6).astype(np.int32)
    return q, t, class_off, q_class, (idx, cnt), cap, gid


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("d", RO.KERNEL_WIDTHS)
def test_rerank_widths_bit_for_bit(dt, d):
    q, t, class_off, q_class, cand, cap, gid = _width_case(dt, d, d)
    for mode in (RO.SAME_CLASS, RO.OTHER_CLASSES):
        for c in (cand, None):
            kw = dict(cand_idx=c[0], cand_cnt=c[1], cap=cap) if c is not None else {}
            want = RO.rerank(q, t, class_off, q_class, mode, t_gid=gid, **kw)
            r = rerank(dt, q, t, class_off, q_class, mode, cand=c, cap=cap, t_gid=gid)
            check(r, want)
            if mode == RO.SAME_CLASS:
                assert r["dist"][1] == 0 and r["pos"][1] == 0
                assert np.isinf(r["dist"][3]) and r["pos"][3] == class_off[2] - 1      # lowest gid of the class
                assert r["dist"][2] > 0                                                 # subnormal squares not flushed


# ---- the list contract ----------------------------------------------------------------------------------------------
def _list_case(dt, d, cap, seed):
    rng = np.random.default_rng(seed)
    n, m = 70, 48
    class_off = np.array([0, 0, 25, 26, 70], dtype=np.int32)            # an empty and a one-row class
    t = (rng.normal(size=(n, d)) * 3).astype(dt)
    t[40:44] = t[30]
    t[[8, 16, 24]] = t[30]
    q = (rng.normal(size=(m, d)) * 3).astype(dt)
    q[:4] = t[30]
    q_class = rng.integers(-1, 5, size=m).astype(np.int32)               # -1 and 4 are invalid
    q_class[:4] = 3
    cnt = rng.integers(0, cap + 2, size=m).astype(np.int32)              # 0 and cap + 1 go to the scan
    cnt[4:8] = (cap, cap + 1, 0, cap)
    q_class[4:8] = 3
    idx = np.zeros((m, cap, 2), dtype=np.int32)
    idx[:, :, 0] = rng.integers(-40, n + 10, size=(m, cap))             # negative starts, bits past n
    idx[:, :, 1] = rng.integers(0, 1 << 32, size=(m, cap), dtype=np.int64).astype(np.uint32).view(np.int32)
    idx[::5, 0, 1] = 0                                                   # empty masks
    if cap > 1:
        idx[1::7, 1] = idx[1::7, 0]                                      # duplicate entries
    idx[8:10, :, 0] = 100                                                # names nothing in range: NaN / -1, no scan
    cnt[8:10] = max(1, cap // 2)
    q_class[8:10] = 2
    if cap >= 4:                                                         # ties over the four 8-lane groups
        for r in range(4):
            idx[r, :4] = [(8, 1), (16, 1), (40, 1), (30, 1)] if r % 2 else [(40, 15), (24, 1), (30, 1), (16, 1)]
            cnt[r] = 4
    gid = np.arange(n)[::-1].astype(np.int32)
    return q, t, class_off, q_class, (idx, cnt), gid


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("d", [5, 37, 128, 200])
def test_rerank_list_contract(dt, d):
    for cap in (1, 3, 4, 64):
        q, t, class_off, q_class, cand, gid = _list_case(dt, d, cap, 100 * d + cap)
        for mode in (RO.SAME_CLASS, RO.OTHER_CLASSES):
            for g in (gid, None):
                want = RO.rerank(q, t, class_off, q_class, mode, cand[0], cand[1], cap, t_gid=g)
                r = rerank(dt, q, t, class_off, q_class, mode, cand=cand, cap=cap, t_gid=g)
                check(r, want)
                assert np.all(r["pos"][8:10] == -1) and np.isnan(r["dist"][8:10]).all()
                bad = (q_class < 0) | (q_class >= 4)
                assert np.all(r["pos"][bad] == -1) and not r["rows"][bad].any()


# ---- the exhaustive scan ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [f32, f64])
def test_rerank_scan_queue_lengths_and_work_reuse(dt):
    rng = np.random.default_rng(21)
    d, n = 24, 40
    class_off = np.array([0, 10, 10, 11, 40], dtype=np.int32)
    t = (rng.normal(size=(n, d)) * 2).astype(dt)
    t[[5, 12, 25, 35, 39]] = t[20]                       # ties that fall into different slices
    for m in (1, 2, 63, 64, 65, 100, 4095, 4096, 4097):
        q = (rng.normal(size=(m, d)) * 2).astype(dt)
        q[::3] = t[20]
        q_class = rng.integers(-1, 5, size=m).astype(np.int32)
        q_class[::4] = (0, 3)[m % 2]                      # OTHER mode for the first and the last class
        work = None
        for mode in (RO.SAME_CLASS, RO.OTHER_CLASSES, RO.SAME_CLASS):
            want = RO.rerank(q, t, class_off, q_class, mode)
            r = rerank(dt, q, t, class_off, q_class, mode, work=work, rows=m < 200)
            check(r, want, rows=m < 200)
            work = r["work"]
        assert want["scanned"] == int(((q_class >= 0) & (q_class < 4)).sum())


@pytest.mark.parametrize("dt", [f32, f64])
def test_rerank_scan_degenerate_ranges(dt):
    rng = np.random.default_rng(5)
    d = 9
    t = rng.normal(size=(12, d)).astype(dt)
    q = rng.normal(size=(7, d)).astype(dt)
    cases = [(np.array([0, 12]), np.zeros(7, np.int32), RO.OTHER_CLASSES),          # n_classes = 1, OTHER: empty
             (np.array([0, 12]), None, RO.SAME_CLASS),                              # q_class NULL
             (np.array([0, 0, 0]), np.array([0, 1, 1, 0, 2, -1, 1], np.int32), RO.SAME_CLASS),   # n = 0
             (np.array([0, 0, 12, 12]), np.array([0, 1, 2, 0, 1, 2, 1], np.int32), RO.OTHER_CLASSES)]
    for class_off, q_class, mode in cases:
        tt = t[:class_off[-1]]
        want = RO.rerank(q, tt, class_off, q_class, mode)
        check(rerank(dt, q, tt, class_off, q_class, mode), want)


@pytest.mark.parametrize("dt", [f32, f64])
def test_rerank_count_overflow_only_then_repeat(dt):
    q, t, class_off, q_class, cand, gid = _list_case(dt, 37, 4, 77)
    want = RO.rerank(q, t, class_off, q_class, RO.SAME_CLASS, cand[0], cand[1], 4, t_gid=gid)
    r = rerank(dt, q, t, class_off, q_class, RO.SAME_CLASS, cand=cand, cap=4, t_gid=gid, count_only=True)
    assert r["wordsw"][0] == want["queued"].sum() > 0 and r["stats"][0] == 0
    listed = ~want["queued"]
    assert np.all(r["pos"][~listed] == np.uint32(0xABABABAB).view(np.int32))
    for k, w in (("dist", "out_dist"), ("pos", "out_pos"), ("gid", "out_gid")):
        assert _same(r[k][listed], want[w][listed])
    r["work"].t[:4].zero_()
    check(rerank(dt, q, t, class_off, q_class, RO.SAME_CLASS, cand=cand, cap=4, t_gid=gid, work=r["work"]), want)


@pytest.mark.parametrize("dt", [f32, f64])
def test_rerank_q_idx_equals_the_gathered_copy(dt):
    q, t, class_off, q_class, cand, gid = _list_case(dt, 130, 4, 8)
    rng = np.random.default_rng(1)
    big = (rng.normal(size=(3 * q.shape[0], q.shape[1])) * 3).astype(dt)
    q_idx = rng.permutation(big.shape[0])[:q.shape[0]].astype(np.int32)
    big[q_idx] = q
    for c in (cand, None):
        a = rerank(dt, big, t, class_off, q_class, RO.OTHER_CLASSES, cand=c, cap=4, t_gid=gid, q_idx=q_idx)
        b = rerank(dt, q, t, class_off, q_class, RO.OTHER_CLASSES, cand=c, cap=4, t_gid=gid)
        for k in ("dist", "pos", "gid", "rows"):
            assert _same(a[k], b[k])
        assert np.array_equal(a["rows"][b["pos"] >= 0], t[b["pos"][b["pos"] >= 0]])


# ---- the fused next stage -------------------------------------------------------------------------------------------
def _query_prep(dt, rows, center):
    torch, _lib, lib = _env()
    m, d = rows.shape
    pitch = lib.tip_pair_pitch(d, 1)
    keep = []
    o = {"pack": Buf(m * pitch * 2), "sqnorm": Buf(m * 4), "rounderr": Buf(m * 4), "row_min": Buf(m * 4),
         "cand_cnt": Buf(m * 4)}
    rc = lib.tip_nn_query_prep(_ptr(keep, rows, dt), _tip(dt), m, d, _ptr(keep, center, np.float32), o["pack"].ptr,
                               o["sqnorm"].ptr, o["rounderr"].ptr, o["row_min"].ptr, o["cand_cnt"].ptr, None, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    return {k: b.get(np.uint16 if k == "pack" else np.uint32, (m, pitch) if k == "pack" else None) for k, b in o.items()}


def _bounded_data(rng, shape, dt):
    """values with |v| in [0.25, 4]: their bf16 squares span less than 2^30, so double partial sums are exact"""
    return (np.sign(rng.normal(size=shape)) * rng.uniform(0.25, 4, size=shape)).astype(dt)


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("d", [5, 37, 100, 128, 200, 1000])
def test_rerank_next_stage_pack_matches_query_prep(dt, d):
    rng = np.random.default_rng(d)
    n, m = 40, 30
    t = _bounded_data(rng, (n, d), dt)
    q = _bounded_data(rng, (m, d), dt)
    class_off = np.array([0, 20, 20, 40], dtype=np.int32)
    q_class = rng.integers(0, 3, size=m).astype(np.int32)       # class 1 is empty: no winner, zero row
    q_class[0] = 7                                               # invalid class
    for center in (None, (rng.uniform(-0.1, 0.1, size=d)).astype(f32)):
        r = rerank(dt, q, t, class_off, q_class, RO.SAME_CLASS, nxt={"center": center})
        want = RO.rerank(q, t, class_off, q_class, RO.SAME_CLASS)
        check(r, want)
        prep = _query_prep(dt, r["rows"], center)
        for k in ("pack", "sqnorm", "rounderr", "row_min", "cand_cnt"):
            assert np.array_equal(r["next_" + k], prep[k]), k
        assert np.array_equal(r["next_pack"], RO.pack_query(want["out_rows"], center))
        assert np.all(r["next_row_min"] == INF32) and np.all(r["next_cand_cnt"] == 0)
        h = RO.bf16_values(r["next_pack"][:, :d])
        c = np.zeros(d, f32) if center is None else center
        fl = ((want["out_rows"] - c.astype(f64)).astype(f32) if dt == f64 else want["out_rows"] - c).astype(f64)
        sq = np.array([f32(math.fsum(row * row)) for row in h])
        assert np.array_equal(r["next_sqnorm"].view(f32), sq)
        exact = np.array([math.sqrt(math.fsum(row * row)) for row in (fl - h)])
        err = r["next_rounderr"].view(f32).astype(f64)
        assert np.all(err >= exact) and np.all(err <= exact * (1 + 2.0 ** -19))
        r2 = rerank(dt, q, t, class_off, q_class, RO.SAME_CLASS, nxt={"center": center, "rounderr": False})
        assert np.array_equal(r2["next_pack"], r["next_pack"]) and np.all(r2["next_row_min"] == INF32)


def _seed_model(ub, nx, q_err, t_rmax, t_err, gamma):
    """seed_row_min_bits() of csrc/common.cuh in float32 (tests/test_window_model.py)"""
    F = f32
    r = F(F(np.sqrt(nx, dtype=F)) + F(t_rmax))
    e = F(F(q_err + F(t_err) + F(1.2e-7) * r) * F(1.00001))
    g = F(gamma * r * r)
    dd = F(F(ub * F(1.000004)) + e)
    return F(F(dd * dd + g) * F(1.000002))


@pytest.mark.parametrize("d", [3, 64, 100, 128, 300])
def test_rerank_next_stage_seeds(d):
    """next_row_min_bits from next_seed_ub: +inf where no row won or the bound is +inf / NaN; otherwise finite, at least
    the seed row's worst-case filter accumulator (the window stays sound), and within 2^-20 of the float32 model."""
    rng = np.random.default_rng(300 + d)
    n, m = 64, 40
    t = (rng.normal(size=(n, d)) * 2).astype(f32)
    q = (rng.normal(size=(m, d)) * 2).astype(f32)
    class_off = np.array([0, 32, 32, 64], dtype=np.int32)
    q_class = rng.integers(0, 3, size=m).astype(np.int32)
    center = t.mean(axis=0).astype(f32)
    partner = (np.arange(n) + 37) % n                           # the row each bound is measured to
    ub = np.array([RO.norms(t[i], t[partner[i]][None])[0] for i in range(n)], dtype=f32)
    ub[::9] = np.inf
    ub[4::9] = np.nan
    tb = RO.bf16_values(RO.pack_query(t, center)[:, :d])
    tfl = (t - center).astype(f64)
    rmax = f32(np.sqrt(np.max(np.sum(tb ** 2, axis=1)))) * f32(1.000001)
    errt = f32(np.sqrt(np.max(np.sum((tfl - tb) ** 2, axis=1)))) * f32(1.000001) * f32(1.000001)
    r = rerank(f32, q, t, class_off, q_class, RO.SAME_CLASS, nxt={"center": center, "seed": (ub, rmax, errt)})
    pos = r["pos"]
    gamma = f32((((d + 15) // 16) * 16 + 32) * 2.0 ** -23)
    seed_s, sqn, qerr = (r[k].view(f32) for k in ("next_row_min", "next_sqnorm", "next_rounderr"))
    seeded = 0
    for i in range(m):
        if pos[i] < 0 or not np.isfinite(ub[pos[i]]):
            assert r["next_row_min"][i] == INF32, i
            continue
        s, nx, qe = seed_s[i], sqn[i], qerr[i]
        model = _seed_model(ub[pos[i]], nx, qe, rmax, errt, gamma)
        assert np.isfinite(s) and s <= model * (1 + 2.0 ** -20), (i, s, model)
        xb = RO.bf16_values(r["next_pack"][i, :d])
        yb = tb[partner[pos[i]]]
        r_ = float(f32(np.sqrt(nx) + rmax))
        worst = float(np.sum(yb ** 2) - 2.0 * (yb @ xb)) + float(gamma) * r_ * r_ + float(nx)
        assert float(s) >= worst, (i, float(s), worst)
        seeded += 1
    assert seeded > 5


# ---- the fused result scatter and tip_dsa_pack_out ---------------------------------------------------------------------
@pytest.mark.parametrize("dt", [f32, f64])
def test_rerank_fused_scatter_equals_pack_out(dt):
    torch, _lib, lib = _env()
    q, t, class_off, q_class, cand, cap, gid = _width_case(dt, 19, 3)
    q = np.concatenate([q, q[:3], np.zeros((1, 19), dt)])
    q_class = np.concatenate([q_class, [9, 0, 0, 0]]).astype(np.int32)   # an invalid class: dist_b NaN
    m = q.shape[0]
    dist_a = np.array([0, 1, 2, 0, np.inf, 3, 5, 0, np.inf, 7], dtype=dt)[:m]
    fgid = np.arange(m, dtype=np.int32) * 3 - 1
    n_total = m + 3
    idx = np.array([3, 0, -1, 2, 5, 4, 1, n_total, 9, 8], dtype=np.int32)[:m]
    fin = {"dist_a": dist_a, "gid": fgid, "idx": idx, "n_total": n_total}
    r = rerank(dt, q, t, class_off, q_class, RO.OTHER_CLASSES, t_gid=gid, fin=fin)
    out = Buf(4 * n_total * 8)
    keep = []
    rc = lib.tip_dsa_pack_out(_ptr(keep, dist_a), _ptr(keep, r["dist"]), _tip(dt), _ptr(keep, fgid), _ptr(keep, idx),
                              m, n_total, out.ptr, _stream())
    torch.cuda.synchronize()
    assert rc == 0 and out.guard_ok()
    sep = out.get(np.float64, (4, n_total))
    assert np.array_equal(r["fin"].view(np.uint64), sep.view(np.uint64))
    want = np.full((4, n_total), np.uint64(0xABABABABABABABAB)).view(np.float64)
    RO.pack_out(dist_a, r["dist"], fgid, idx, n_total, want)
    assert _same(sep, want)
    named = np.zeros(n_total, bool)
    named[idx[(idx >= 0) & (idx < n_total)]] = True
    assert np.all(sep[:, ~named].view(np.uint64) == 0xABABABABABABABAB) and (~named).sum() >= 3
    ratio = sep[3, idx[[0, 3, 4, 6]]]                          # 0/x, 0/0 or x/0, inf/x, x/inf as NumPy gives them
    with np.errstate(divide="ignore", invalid="ignore"):
        assert _same(ratio, (dist_a[[0, 3, 4, 6]] / r["dist"][[0, 3, 4, 6]]).astype(f64))


@pytest.mark.parametrize("dt", [f32, f64])
def test_pack_out_numpy_division(dt):
    torch, _lib, lib = _env()
    a = np.array([0, 1, np.inf, 2, 0, 3, np.nan], dtype=dt)
    b = np.array([0, 0, np.inf, np.inf, 5, np.nan, 1], dtype=dt)
    gid = np.arange(7, dtype=np.int32)
    out = Buf(4 * 7 * 8)
    keep = []
    assert lib.tip_dsa_pack_out(_ptr(keep, a), _ptr(keep, b), _tip(dt), _ptr(keep, gid), None, 7, 7, out.ptr,
                                _stream()) == 0
    torch.cuda.synchronize()
    got = out.get(np.float64, (4, 7))
    assert np.isnan(got[3, [0, 2, 5, 6]]).all() and got[3, 1] == np.inf and got[3, 3] == 0 and got[3, 4] == 0
    assert _same(got, RO.pack_out(a, b, gid, None, 7, np.zeros((4, 7))))


# ---- tip_gather_rows -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row_bytes,offset,m", [(48, 0, 200000), (16, 0, 5), (12, 0, 9000), (28, 4, 300),
                                                (64, 4, 1000), (4100, 0, 40)])
def test_gather_rows(row_bytes, offset, m):
    torch, _lib, lib = _env()
    rng = np.random.default_rng(row_bytes + m)
    n = 257
    src = rng.integers(0, 256, size=n * row_bytes + offset, dtype=np.uint8)
    pos = rng.integers(-2, n, size=m).astype(np.int32)
    d_src = _dev(src)
    out = Buf(m * row_bytes + offset)
    keep = []
    rc = lib.tip_gather_rows(d_src.data_ptr() + offset, row_bytes, _ptr(keep, pos), m, out.ptr + offset, _stream())
    torch.cuda.synchronize()
    assert rc == 0 and out.guard_ok()
    rows = src[offset:].reshape(n, row_bytes)
    want = np.where((pos >= 0)[:, None], rows[np.maximum(pos, 0)], 0)
    got = out.get(np.uint8)
    assert np.all(got[:offset] == FILL) and np.array_equal(got[offset:].reshape(m, row_bytes), want)


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_rerank_argument_checks_launch_nothing():
    torch, _lib, lib = _env()
    keep = []
    q = _ptr(keep, np.zeros((4, 8), f32))
    off = _ptr(keep, np.array([0, 4], np.int32))
    idx, cnt = _ptr(keep, np.zeros((4, 2, 2), np.int32)), _ptr(keep, np.ones(4, np.int32))
    outs = [Buf(64) for _ in range(8)]
    work = Buf(lib.tip_nn_rerank_work_bytes(4, 0), zero=True)

    def call(m=4, cand=(None, None), cap=2, mode=0, ex=None, nxt=False, rounderr=True):
        e = ex or _lib.RerankExtras()
        pk = [outs[3].ptr, outs[4].ptr, outs[5].ptr if rounderr else None, outs[6].ptr, outs[7].ptr] if nxt else [None] * 5
        return lib.tip_nn_rerank(q, q, 0, m, 4, 8, cand[0], cand[1], cap, None, off, 1, mode, None, outs[0].ptr,
                                 outs[1].ptr, None, None, work.ptr, None, None, pk[0], pk[1], pk[2], pk[3], pk[4],
                                 C.byref(e), _stream())

    seeds = _lib.RerankExtras()
    seeds.next_seed_ub = _ptr(keep, np.zeros(4, f32))
    fin = _lib.RerankExtras()
    fin.fin_out = outs[2].ptr
    only = _lib.RerankExtras()
    only.count_overflow_only = 1
    torch.cuda.synchronize()
    before = lib.tip_launch_count()
    assert call(ex=seeds, nxt=True, rounderr=False) == -1
    assert call(ex=fin) == -1
    assert call(ex=only) == -1
    assert call(mode=2) == -1
    assert call(cand=(idx, cnt), cap=0) == -1
    assert call(m=0) == 0
    assert lib.tip_launch_count() == before
    torch.cuda.synchronize()
    assert all(b.get(np.uint8).tolist() == [FILL] * 64 for b in outs)


# ---- the hand-over kernels of the sharded search ---------------------------------------------------------------------
def _winner_queries(dt, comm, gdist, ggid, train, center, m=None):
    """tip_shard_winner_queries: from the reduced (gdist, ggid), or (comm, gdist = ggid = None) from the records of
    the last push."""
    torch, _lib, lib = _env()
    m = len(ggid) if m is None else m
    n_full, d = train.shape
    es = np.dtype(dt).itemsize
    pitch = lib.tip_pair_pitch(d, 1)
    keep = []
    o = {"dist": Buf(m * es), "gid": Buf(m * 4), "rows": Buf(m * d * es), "pack": Buf(m * pitch * 2),
         "sqnorm": Buf(m * 4), "rounderr": Buf(m * 4), "row_min": Buf(m * 4), "cand_cnt": Buf(m * 4)}
    rc = lib.tip_shard_winner_queries(comm, _ptr(keep, gdist, dt), _ptr(keep, ggid, np.int32), _tip(dt), m, d,
                                      _ptr(keep, train), n_full, _ptr(keep, center, np.float32), o["dist"].ptr,
                                      o["gid"].ptr, o["rows"].ptr, o["pack"].ptr, o["sqnorm"].ptr, o["rounderr"].ptr,
                                      o["row_min"].ptr, o["cand_cnt"].ptr, _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.tip_last_error()
    assert all(b.guard_ok() for b in o.values())
    return {"dist": o["dist"].get(dt), "gid": o["gid"].get(np.int32), "rows": o["rows"].get(dt, (m, d)),
            **{k: o[k].get(np.uint16 if k == "pack" else np.uint32, (m, pitch) if k == "pack" else None)
               for k in ("pack", "sqnorm", "rounderr", "row_min", "cand_cnt")}}


def _winner_case(dt, d=21):
    rng = np.random.default_rng(d)
    train = (rng.normal(size=(30, d)) * 2).astype(dt)
    gdist = np.array([0.5, 2, np.nan, 1, np.inf, np.inf, 0, 3], dtype=dt)
    ggid = np.array([3, 29, 4, -1, 7, -1, 30, 0], dtype=np.int32)
    keep = np.isfinite(gdist) | np.isinf(gdist)
    keep &= (ggid >= 0) & (ggid < 30)
    want_dist = np.where(keep, gdist, np.nan).astype(dt)
    want_gid = np.where(keep, ggid, -1).astype(np.int32)
    want_rows = np.where(keep[:, None], train[np.maximum(ggid, 0) % 30], 0).astype(dt)
    return train, gdist, ggid, want_dist, want_gid, want_rows, rng.uniform(-0.5, 0.5, d).astype(f32)


def _check_winners(dt, got, want_dist, want_gid, want_rows, center):
    assert _same(got["dist"], want_dist) and np.array_equal(got["gid"], want_gid)
    assert _same(got["rows"], want_rows)
    prep = _query_prep(dt, want_rows, center)
    for k in ("pack", "sqnorm", "rounderr", "row_min", "cand_cnt"):
        assert np.array_equal(got[k], prep[k]), k


@pytest.mark.parametrize("dt", [f32, f64])
def test_shard_winner_queries_keep_inf_and_drop_none(dt):
    train, gdist, ggid, wd, wg, wr, center = _winner_case(dt)
    assert np.isinf(wd[4]) and wg[4] == 7                        # a real +inf distance keeps its winner
    got = _winner_queries(dt, None, gdist, ggid, train, center)
    _check_winners(dt, got, wd, wg, wr, center)


def test_comm_exchange_world1_keeps_inf():
    """tip_comm_* at world 1: the only flag is this rank's own, raised by the push issued before each consumer on
    the same stream, so no wait can spin.  Three exchanges use both parities of the double-buffered slots."""
    torch, _lib, lib = _env()
    local = C.c_void_p(0)
    handle = (C.c_ubyte * 64)()
    cap = 64
    if lib.tip_comm_alloc(1, cap, C.byref(local), handle) != 0:
        pytest.skip("tip_comm_alloc: " + lib.tip_last_error().decode(errors="replace"))
    comm = C.c_void_p(0)
    try:
        assert lib.tip_comm_open(0, 1, local, handle, cap, C.byref(comm)) == 0, lib.tip_last_error()
        keep = []
        for it in range(3):
            for dt in (f32, f64):
                train, gdist, ggid, wd, wg, wr, center = _winner_case(dt, 21 + it)
                assert lib.tip_comm_push_nn(comm, _ptr(keep, gdist, dt), _tip(dt), _ptr(keep, ggid, np.int32),
                                            len(gdist), _stream()) == 0
                mn = Buf(len(gdist) * np.dtype(dt).itemsize)
                assert lib.tip_comm_min(comm, _tip(dt), len(gdist), mn.ptr, _stream()) == 0
                torch.cuda.synchronize()
                got = mn.get(dt)
                assert _same(got, gdist)                         # NaN stays NaN, +inf stays +inf
                assert np.isinf(got[4]) and np.isinf(got[5]) and np.isnan(got[2])
                assert lib.tip_comm_push_nn(comm, _ptr(keep, gdist, dt), _tip(dt), _ptr(keep, ggid, np.int32),
                                            len(gdist), _stream()) == 0
                got = _winner_queries(dt, comm, None, None, train, center, m=len(gdist))
                ref = _winner_queries(dt, None, gdist, ggid, train, center)
                _check_winners(dt, ref, wd, wg, wr, center)
                for k in ref:
                    assert np.array_equal(got[k].view(np.uint8), ref[k].view(np.uint8)), k
            pm = np.array([0.5, -np.inf, 3e38, -2], dtype=f32)
            ps = np.array([1.25, 0, 7, 3e-39], dtype=f32)
            assert lib.tip_comm_push_lse(comm, _ptr(keep, pm), _ptr(keep, ps), 4, _stream()) == 0
            om, os_ = Buf(16), Buf(32)
            assert lib.tip_comm_lse(comm, 4, om.ptr, os_.ptr, _stream()) == 0
            torch.cuda.synchronize()
            assert np.array_equal(om.get(f32), pm)
            assert np.array_equal(os_.get(f64), np.where(pm == -np.inf, 0.0, ps.astype(f64)))
    finally:
        torch.cuda.synchronize()
        lib.tip_comm_close(comm)
        lib.tip_comm_free_local(local)


# ---- DSA end to end on traces whose squares overflow ----------------------------------------------------------------
@pytest.mark.parametrize("dt", [f32, f64])
def test_dsa_with_overflowing_distances_matches_numpy(dt):
    """Rows at ~1e20 (float32: their squared differences overflow; float64: 1e300, beyond float32's range) mixed with
    ordinary ones, and a query equal to a huge row: the single-GPU DSA gives NumPy's bits, +inf distances and NaN
    ratios included.  The packed bf16 rows have no finite bound, so the filter stays off and every query takes the
    exact scan (float64 traces like these used to be rejected by tip_nn_filter's t_errmax check)."""
    from simple_tip_b200.core.surprise import DSA

    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(600, 80, 24, 3, seed=17, dtype=dt)
    huge = 1e20 if dt == f32 else 1e300
    xtr[::7] = huge * (1 + np.random.default_rng(0).random((xtr[::7].shape[0], 24))).astype(dt)
    xte[:10] = -huge
    xte[10] = xtr[7]
    pte[10] = ytr[7]
    want = np_oracle.dsa_oracle(xtr, ytr, xte, pte)
    assert np.isinf(want["dist_a"]).any()
    sa = DSA(xtr, ytr)
    got = sa(xte, pte)
    assert _same(sa.last_dist_a, want["dist_a"]) and _same(sa.last_dist_b, want["dist_b"])
    assert np.array_equal(sa.last_winner_index, want["idx_a"])
    assert _same(got, want["dsa"])
    assert not sa._engine.filter_ok
    assert sa._engine.stats.cpu().numpy()[0] >= xte.shape[0]          # the queries took the exact scan
