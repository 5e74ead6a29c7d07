"""The filter checker of oracle/filter_oracle.py has teeth: on hand-made accumulators and candidate lists it accepts the
lists an exact filter emits, and rejects each way a kernel can lose or invent a candidate (a required column dropped,
a row minimum taken without the range's last tile, a chunk emitted twice, a bit past the span, a bit under the
excluded class).  And the two threshold bounds it uses enclose a float32 emulation of nn_threshold()."""
import numpy as np
import pytest

pytest.importorskip("torch")

from oracle import filter_oracle as FO  # noqa: E402

F32 = np.float32
D = 20                                  # k16 = 3
N = 300
CLASS_OFF = np.array([0, 100, 190, N], dtype=np.int64)     # class starts that are not multiples of 32
Q_CLASS = np.array([0, 0, 1, 1, 2], dtype=np.int32)
# rows 0-1: one span over every column; rows 2-3: a flagged item that starts and ends mid-chunk (its rows skip their
# own class 1 = [100, 190)) and a second item for the rest; row 4: no item
ITEMS = np.array([[0, 2, 0, N, 0, 0],
                  [2, 2, 5, 250, 0, 1],
                  [2, 2, 250, 250, 0, 0],
                  [2, 2, 250, N, 0, 1]], dtype=np.int32)
CAP = 16


def _nn_threshold(s, nx, e2, g, fused_tail=True):
    """nn_threshold() in float32 with a correctly rounded sqrt in place of sqrt.approx; fmaf(r, r, g) as one rounding,
    and thr + |thr| 1e-6 fused (as nvcc contracts it) or not."""
    root = F32(np.sqrt(F32(F32(s) + F32(g)), dtype=F32))
    r = F32(F32(root + F32(e2)) * F32(1.00004))
    thr = F32(F32(np.float64(r) * np.float64(r) + np.float64(F32(g))) - F32(nx))
    t = F32(thr + np.float64(abs(thr)) * np.float64(F32(1e-6))) if fused_tail else F32(thr + F32(abs(thr) * F32(1e-6)))
    return F32(t + F32(1e-30))


def _case():
    """Accumulators a = d^2 - |x|^2 for |x|^2 = 100: a few near rows per query, rows planted just inside and just
    outside the window, the rest far away."""
    rng = np.random.default_rng(5)
    m = Q_CLASS.shape[0]
    nx = np.full(m, 100.0, dtype=F32)
    win = FO.window(nx, None, 20.0, 0.0, D)
    d2 = rng.uniform(30.0, 400.0, size=(m, N))
    for i in range(m):
        near = rng.choice(np.flatnonzero(FO.row_ranges(m, N, ITEMS, Q_CLASS, CLASS_OFF)[0][i]), size=8, replace=False) \
            if i < 4 else rng.choice(N, size=8, replace=False)
        d2[i, near[0]] = 4.0                           # the argmin
        d2[i, near[1]] = 4.0                           # an exact tie with it
        s = float(F32(4.0 + 0.0))
        t_lo = float(FO.threshold_lo(F32(s), nx[i], win.e2_lo[i], win.g[i])) + float(nx[i])
        for k, f in enumerate((0.2, 0.5, 0.9, 1.1, 1.5, 3.0)):   # fractions of the way to the window's edge
            d2[i, near[2 + k]] = 4.0 + f * (t_lo - float(win.g[i]) - 4.0)
    a = d2 - 100.0
    return a, win


def _emit(a, win, inr, items, row_min):
    """What an exact filter writes: per item and 32-column chunk of its span (chunks start at col0 + 32 k), the columns
    of the row's range inside nn_threshold(row_min)."""
    m, n = a.shape
    idx = np.zeros((m, CAP, 2), dtype=np.int32)
    cnt = np.zeros(m, dtype=np.int32)
    for r0, nr, c0, c1, _, _ in items:
        for i in range(r0, r0 + nr):
            thr = float(_nn_threshold(F32(np.uint32(row_min[i]).view(F32)), win.nx[i], win.e2_lo[i], win.g[i]))
            for col in range(c0, c1, 32):
                cols = np.arange(col, min(col + 32, c1))
                ok = inr[i, cols] & (a[i, cols] <= thr)
                mask = int(np.sum((ok.astype(np.uint64)) << (cols - col).astype(np.uint64)))
                if mask:
                    if cnt[i] < CAP:
                        idx[i, cnt[i]] = (col, np.uint32(mask).view(np.int32))
                    cnt[i] += 1
    return idx, cnt


def _run(a, win, idx, cnt, row_min, items=ITEMS):
    inr, owner, times = FO.row_ranges(a.shape[0], a.shape[1], items, Q_CLASS, CLASS_OFF)
    return FO.check(a, np.zeros_like(a), win, inr, owner, row_min, idx, cnt, CAP, times=times)


def _row_min(a, win, inr):
    out = np.full(a.shape[0], FO.INF_BITS, dtype=np.uint32)
    for i in range(a.shape[0]):
        if inr[i].any():
            out[i] = np.float32(max(a[i, inr[i]].min() + float(win.nx[i]), 0.0)).view(np.uint32)
    return out


@pytest.fixture(scope="module")
def clean():
    a, win = _case()
    inr, _, _ = FO.row_ranges(a.shape[0], a.shape[1], ITEMS, Q_CLASS, CLASS_OFF)
    row_min = _row_min(a, win, inr)
    idx, cnt = _emit(a, win, inr, ITEMS, row_min)
    return a, win, inr, row_min, idx, cnt


def _kinds(rep):
    return {f["kind"] for f in rep.findings}


def test_exact_lists_pass_and_the_check_is_not_vacuous(clean):
    a, win, inr, row_min, idx, cnt = clean
    rep = _run(a, win, idx, cnt, row_min)
    assert not rep.findings, rep.summary()
    assert rep.checked_rows == 4 and rep.overflowed == 0
    assert rep.required_extra >= 4 * 3           # the tie and the 0.2 / 0.5 rows (0.9 sits at the rounding's edge)
    assert rep.outside > 0
    assert rep.rowmin_frac == 0.0
    # the uncovered row keeps the prepared state
    assert row_min[4] == FO.INF_BITS and cnt[4] == 0


def test_rejects_a_missing_required_column(clean):
    a, win, inr, row_min, idx, cnt = clean
    idx = idx.copy()
    i = 0
    j_min = int(np.flatnonzero(inr[i])[np.argmin(a[i, inr[i]])])
    ties = np.flatnonzero(inr[i] & (a[i] == a[i, j_min]))
    j = int(ties[ties != j_min][0])                                      # the tied row: required beyond the argmin
    for k in range(cnt[i]):
        col, mask = idx[i, k]
        if col <= j < col + 32 and ((int(mask) & 0xFFFFFFFF) >> (j - col)) & 1:
            idx[i, k, 1] = np.uint32(int(mask) & 0xFFFFFFFF & ~(1 << (j - col))).view(np.int32)
    rep = _run(a, win, idx, cnt, row_min)
    assert any(f["kind"] == "required column missing from the list" and f["col"] == j for f in rep.findings), \
        rep.summary()


def test_rejects_a_row_min_without_the_ranges_last_tile(clean):
    a, win, inr, row_min, idx, cnt = clean
    a = a.copy()
    i = 1
    a[i, N - 3] = a[i, inr[i]].min() - 50.0                           # the row's minimum, in the span's last tile
    inr_wo = inr.copy()
    inr_wo[i, (N - 1) // 128 * 128:] = False
    wrong = _row_min(a, win, inr_wo)
    rep = _run(a, win, idx, cnt, wrong)
    assert any(f["kind"] == "row_min off the range's minimum" and f["row"] == i for f in rep.findings), rep.summary()
    assert rep.rowmin_frac > 1.0


def test_rejects_a_duplicated_chunk(clean):
    a, win, inr, row_min, idx, cnt = clean
    idx, cnt = idx.copy(), cnt.copy()
    i = 2
    idx[i, cnt[i]] = idx[i, 0]
    cnt[i] += 1
    rep = _run(a, win, idx, cnt, row_min)
    assert "column admitted twice" in _kinds(rep), rep.summary()


def test_rejects_a_bit_past_the_span(clean):
    a, win, inr, row_min, idx, cnt = clean
    idx, cnt = idx.copy(), cnt.copy()
    i = 0
    idx[i, cnt[i]] = (N - 20, np.uint32(1 << 25).view(np.int32))     # column N + 5
    cnt[i] += 1
    rep = _run(a, win, idx, cnt, row_min)
    assert "bit outside the train rows" in _kinds(rep), rep.summary()
    # and one inside the train rows but before the flagged item's first column
    idx[i, cnt[i] - 1] = idx[i, 0]
    i = 3
    idx[i, cnt[i]] = (0, np.uint32(1 << 2).view(np.int32))            # column 2 < col0 = 5
    cnt[i] += 1
    rep = _run(a, win, idx, cnt, row_min)
    assert any(f["kind"] == "bit outside the row's range" and (f["row"], f["col"]) == (3, 2) for f in rep.findings), \
        rep.summary()


def test_rejects_a_bit_under_the_excluded_class(clean):
    a, win, inr, row_min, idx, cnt = clean
    idx, cnt = idx.copy(), cnt.copy()
    i = 2                                                             # class 1: columns [100, 190) are excluded
    idx[i, cnt[i]] = (165, np.uint32(1 << 24).view(np.int32))          # column 189, the class's last row
    cnt[i] += 1
    rep = _run(a, win, idx, cnt, row_min)
    assert any(f["kind"] == "bit outside the row's range" and (f["row"], f["col"]) == (2, 189) for f in rep.findings), \
        rep.summary()
    # the same column is fine for a row of another class scanning it
    assert inr[0, 189]


def test_rejects_a_work_list_that_scans_a_pair_twice(clean):
    a, win, inr, row_min, idx, cnt = clean
    rep = _run(a, win, idx, cnt, row_min, items=np.vstack([ITEMS, [[0, 1, 30, 40, 0, 0]]]).astype(np.int32))
    assert "pair scanned by more than one item (the work list breaks its contract)" in _kinds(rep)


def test_threshold_bounds_enclose_the_kernels_formula():
    rng = np.random.default_rng(9)
    n = 20000
    s = np.exp(rng.uniform(np.log(1e-8), np.log(1e8), n))
    nx = np.exp(rng.uniform(np.log(1e-6), np.log(1e8), n))
    e2 = np.exp(rng.uniform(np.log(1e-9), np.log(1e3), n))
    g = np.exp(rng.uniform(np.log(1e-12), np.log(1e4), n))
    cases = list(zip(s, nx, e2, g))
    ext = [0.0, 1e-30, 1e-7, 1.0, 3.0e4, 1e12, 1e30]
    cases += [(a, b, c, d) for a in ext for b in ext[:-1] for c in (0.0, 1e-6, 0.5, 1e3) for d in (0.0, 1e-9, 7.0)]
    for s_, nx_, e2_, g_ in cases:
        s_, nx_, e2_, g_ = F32(s_), F32(nx_), F32(e2_), F32(g_)
        lo = float(FO.threshold_lo(s_, nx_, e2_, g_))
        hi = float(FO.threshold_hi(float(s_), float(nx_), float(e2_), float(g_)))
        for fused in (True, False):
            k = float(_nn_threshold(s_, nx_, e2_, g_, fused))
            assert lo <= k <= hi, (float(s_), float(nx_), float(e2_), float(g_), fused, lo, k, hi)
