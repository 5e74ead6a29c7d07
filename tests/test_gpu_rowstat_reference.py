"""The softmax row-statistic kernels (`rowstat_small_kernel`, `rowstat_wide_kernel`) and the vote kernels
(`vote_add_kernel`, `vote_finish_kernel`) of csrc/simple.cu against NumPy, at the edges where their launch changes.

* The entropy is checked in its own summation order, bit for bit.  Each element's term q*log2(q) comes from the kernel
  itself (a C = 1 row's entropy is -term), and the reference is NumPy's pairwise `-np.sum(T, axis=1)` over those
  terms, summed the way `np_oracle.deepgini_oracle` sums p*p.  The term is checked on its own against a long-double
  q*log2(q).
* DeepGini, max softmax, PCS and every prediction are bit-exact against oracle/np_oracle.py and
  oracle/quantifier_oracle.py at the widths where the route changes, over more than one grid wave of rows, and on
  crafted rows: ties across the wide kernel's lanes, a repeated maximum, infinities.
* Rows with NaN follow NumPy: the prediction is np.argmax's (the first NaN), max softmax and PCS are NaN, and a sample
  votes for its np.argmax.

Routes (launch_rowstat): a row goes to the thread-per-row kernel while 128 * (c + 1) * sizeof(T) <= 96 KiB, else to
the warp-per-row kernel, which stages GINI / ENTROPY rows in shared memory up to c = 4096 and refuses them above
kGiniMaxLeaves * 64 = 65536.  One grid wave is SMs * 8 blocks of 128 rows (small) or SMs * 16 blocks of 4 rows (wide).
Votes (tip_vote_add): one thread per sampled row up to c = 32, a warp above; rows_per_block = max(1, min(256 // S,
12288 // c)) rows count in shared memory while rows_per_block * c <= 12288, in global memory otherwise."""
import numpy as np
import pytest

from oracle import np_oracle
from oracle import quantifier_oracle as QO

pytestmark = pytest.mark.gpu

SMALL_SMEM = 96 * 1024
STAGE_ELEMS = 4096
MAX_SUM_C = 1024 * 64
VOTE_THREAD_C = 32
VOTE_SMEM_INTS = 12 * 1024

WIDTHS = [1, 2, 7, 8, 9, 15, 16, 17, 95, 96, 127, 128, 129, 136, 191, 192, 255, 256, 257, 4096, 4097, 65536]
DTYPES = [np.float32, np.float64]


def _torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def sms():
    torch = _torch()
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _route(c, dt):
    if 128 * (c + 1) * np.dtype(dt).itemsize <= SMALL_SMEM:
        return "small"
    return "wide, staged" if c <= STAGE_ELEMS else "wide"


def _vote_route(s, c):
    rpb = max(1, min(256 // s, VOTE_SMEM_INTS // c))
    return rpb, ("thread" if c <= VOTE_THREAD_C else "warp"), ("shared" if rpb * c <= VOTE_SMEM_INTS else "global")


def _diff_rows(got, want):
    """Indices where got and want differ: NaN must meet NaN, every other value must have the same bits."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    u = {4: np.uint32, 8: np.uint64}[got.itemsize]
    same = np.where(gn | wn, gn & wn, got.view(u) == want.view(u))
    return np.flatnonzero(~same)


def _rows(n, c, dt, seed):
    """Dirichlet(0.3) rows, a third of every seventh row exactly zero."""
    rng = np.random.default_rng(seed)
    p = rng.dirichlet(np.full(c, 0.3), size=n)
    p[::7, : c // 3] = 0
    return p.astype(dt)


def _crafted(c, dt, seed):
    """Rows whose maxima sit where the wide kernel's lanes (element k in lane k % 32) must merge them."""
    rng = np.random.default_rng(seed)
    out = []

    def plant(idx, val=0.5):
        if len(set(idx)) == len(idx) and max(idx) < c:
            r = rng.uniform(0, 0.1, size=c)
            r[list(idx)] = val
            out.append(r)

    plant([c // 2, c // 2 + 1])                 # top two equal in neighbouring lanes
    plant([3, 35])                              # top two equal in one lane, k and k + 32
    plant([31, 32])                             # a tie: the lower index is in the higher lane
    plant([1, 64])
    plant([c - 2, c - 1])
    plant([0, c // 3, c - 1])                   # the maximum three times
    plant([40, 7, 70])
    plant([c // 2, c - 1], np.inf)              # two +inf: PCS is inf - inf = NaN
    plant([0], np.inf)
    out.append(np.full(c, -np.inf))             # all -inf: PCS is NaN, DeepGini -inf
    r = rng.uniform(0, 0.1, size=c)
    r[: c - 1] = -np.inf                        # -inf but for the last column
    out.append(r)
    out.append(np.full(c, 1.0 / c))             # every class tied
    return np.array(out, dtype=dt).reshape(-1, c)


def _terms(p_dev):
    """The kernel's own entropy_term(q) of every element of p_dev [n, c]: a one-class row's entropy is -term."""
    from simple_tip_b200.core.quantifiers import SoftmaxEntropy

    _, e = SoftmaxEntropy.calculate(p_dev.reshape(-1, 1))
    return np.ascontiguousarray(-e.reshape(p_dev.shape))


def _check_all(p, p_dev, label):
    """Every statistic and prediction of p (on the device as p_dev) against NumPy."""
    from simple_tip_b200.core.deepgini import DeepGini
    from simple_tip_b200.core.quantifiers import MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy

    want_pred = np.argmax(p, axis=1)
    runs = [(DeepGini, np_oracle.deepgini_oracle), (MaxSoftmax, QO.max_softmax)]
    if p.shape[1] >= 2:
        runs.append((PredictionConfidenceScore, QO.pcs))
    for cls, oracle in runs:
        pred, val = cls.calculate(p_dev)
        bad = np.flatnonzero(pred != want_pred)
        assert bad.size == 0, (label, cls.__name__, "pred", bad[:8], pred[bad[:8]], want_pred[bad[:8]])
        want = oracle(p)[1]
        bad = _diff_rows(val, want)
        assert bad.size == 0, (label, cls.__name__, bad[:8], val[bad[:8]], want[bad[:8]])
    t = _terms(p_dev)
    pred, ent = SoftmaxEntropy.calculate(p_dev)
    bad = np.flatnonzero(pred != want_pred)
    assert bad.size == 0, (label, "SoftmaxEntropy pred", bad[:8])
    bad = _diff_rows(ent, -np.sum(t, axis=1))
    assert bad.size == 0, (label, "entropy off NumPy's pairwise sum of its terms", bad[:8])


# ---------------------------------------------------------------------------------------------------------------
# a. The entropy's term, and its sum in NumPy's order
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
def test_entropy_term_against_long_double(dt):
    """entropy_term(q) = q * log2(q), q = p with 0 -> 1e-20: the log2 within an ulp of the dtype, plus the one rounding
    of the product.  float32's log2 is float64 log2 rounded once, and its term is NumPy's float32 product with that
    log2.  float64's is CUDA's log2, documented to one ulp; the test allows two."""
    torch = _torch()
    rng = np.random.default_rng(1)
    tiny = np.finfo(dt).tiny
    p = np.concatenate([
        10.0 ** rng.uniform(-30, 0, size=400_000),                    # log-uniform over the softmax range
        rng.uniform(0, 1, size=400_000),
        1 - rng.uniform(0, 1e-6, size=50_000),                        # log2 near 0
        np.ldexp(1.0, np.arange(-100, 1)),                             # exact powers of two
        [0.0, -0.0, 1.0, tiny, np.nextafter(dt(1), dt(0)), 1e-20, 0.5, 1.0 / 3]]).astype(dt)
    t = _terms(torch.from_numpy(p.reshape(-1, 1)).cuda()).ravel()
    q = np.where(p == 0, dt(1e-20), p)
    ql = q.astype(np.longdouble)
    exact = ql * np.log2(ql)
    log_ulp = np.abs(ql) * np.spacing(np.abs(np.log2(ql).astype(dt))).astype(np.longdouble)    # |q| * ulp(log2 q)
    half_ulp = np.spacing(np.abs(t)).astype(np.longdouble) / 2
    err = np.abs(t.astype(np.longdouble) - exact)
    log_ulps = float(np.max((err - half_ulp) / log_ulp))            # a lower bound of the worst log2 error, in ulps
    print(f"\n{np.dtype(dt).name}: the worst term's log2 is off by at least {log_ulps:.3f} ulp ({p.size} values)")
    allowed = 1 if dt == np.float32 else 2
    bad = err > allowed * log_ulp + half_ulp
    assert not bad.any(), (q[bad][:8], t[bad][:8])
    if dt == np.float32:
        want = q * np.log2(q.astype(np.float64)).astype(np.float32)
        bad = np.flatnonzero(t != want)
        assert bad.size == 0, ("float32 term is not float64 log2 rounded once", q[bad[:8]], t[bad[:8]], want[bad[:8]])
    assert np.all(t[p == 0] == t[p == dt(1e-20)][0])           # an exact zero is read as 1e-20


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
def test_entropy_sums_in_numpys_order(dt, c):
    torch = _torch()
    from simple_tip_b200.core.quantifiers import SoftmaxEntropy

    n = 257 if c < 4096 else (67 if c < 65536 else 9)
    p = _rows(n, c, dt, seed=c)
    p_dev = torch.from_numpy(p).cuda()
    t = _terms(p_dev)
    assert t.dtype == dt and t.flags.c_contiguous
    pred, ent = SoftmaxEntropy.calculate(p_dev)
    want = -np.sum(t, axis=1)
    bad = _diff_rows(ent, want)
    assert bad.size == 0, (_route(c, dt), bad[:8], ent[bad[:8]], want[bad[:8]])
    assert np.array_equal(pred, np.argmax(p, axis=1))
    # teeth: summed in another order the same terms give other bits, so a kernel that changed its order would fail
    seq = -np.cumsum(t, axis=1)[:, -1]
    share = float(np.mean(seq != want))
    print(f"\nc = {c} {np.dtype(dt).name} ({_route(c, dt)}): sequential sum differs on {share:.0%} of rows")
    if c >= 9:
        assert share >= 0.1, share


# ---------------------------------------------------------------------------------------------------------------
# b. All four statistics and the predictions at the route edges
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
def test_statistics_at_the_route_edges(dt, c):
    torch = _torch()
    n = 257 if c < 4096 else (67 if c < 65536 else 9)
    craft = _crafted(c, dt, seed=c)
    p = np.concatenate([craft, _rows(n, c, dt, seed=c + 1)])
    p_dev = torch.from_numpy(p).cuda()
    _check_all(p, p_dev, (c, np.dtype(dt).name, _route(c, dt)))
    print(f"\nc = {c} {np.dtype(dt).name}: {p.shape[0]} rows ({_route(c, dt)}), {len(craft)} crafted")


def test_crafted_rows_hold_what_they_claim():
    """The crafted rows put the maximum where the lanes must merge it (pure NumPy)."""
    p = _crafted(300, np.float32, seed=0)
    assert list(np.argmax(p[:7], axis=1)) == [150, 3, 31, 1, 298, 0, 7]
    pcs = QO.pcs(p)[1]
    assert np.all(pcs[:7] == 0) and pcs[11] == 0
    assert np.isnan(pcs[7]) and np.isnan(pcs[9]) and pcs[8] == np.inf and pcs[10] == np.inf


@pytest.mark.parametrize("dt", DTYPES)
def test_widths_past_the_tree_are_refused_before_any_launch(dt):
    torch = _torch()
    from simple_tip_b200 import _lib
    from simple_tip_b200.core.deepgini import DeepGini
    from simple_tip_b200.core.quantifiers import MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy

    c = MAX_SUM_C + 1
    p = _rows(5, c, dt, seed=3)
    p_dev = torch.from_numpy(p).cuda()
    for cls in (DeepGini, SoftmaxEntropy):
        before = _lib.launch_count()
        with pytest.raises(_lib.TipError, match="row too wide"):
            cls.calculate(p_dev)
        assert _lib.launch_count() == before, cls.__name__
    for cls, oracle in ((MaxSoftmax, QO.max_softmax), (PredictionConfidenceScore, QO.pcs)):
        pred, val = cls.calculate(p_dev)                 # no sum, no tree: these run at any width
        assert np.array_equal(pred, np.argmax(p, axis=1)) and _diff_rows(val, oracle(p)[1]).size == 0


@pytest.mark.parametrize("c,dt", [(7, np.float32), (95, np.float64), (192, np.float32), (96, np.float64),
                                  (4097, np.float32)])
def test_more_than_one_grid_wave(sms, c, dt):
    """2.2 grid waves of rows and a partial last block: every row through the grid-stride loop's later passes."""
    torch = _torch()
    route = _route(c, dt)
    wave = sms * 8 * 128 if route == "small" else sms * 16 * 4
    block = 128 if route == "small" else 4
    n = 2 * wave + wave // 5 // block * block + block // 2 + 1
    assert n > 2 * wave and n % block != 0
    p = _rows(n, c, dt, seed=c)
    craft = _crafted(c, dt, seed=c)
    at = np.linspace(0, n - len(craft), 5).astype(int)
    for a in at:                                              # crafted rows in the first, later and last blocks
        p[a:a + len(craft)] = craft
    p[-1] = craft[2]
    p_dev = torch.from_numpy(p).cuda()
    _check_all(p, p_dev, (c, np.dtype(dt).name, route, n))
    print(f"\nc = {c} {np.dtype(dt).name} ({route}): {n} rows = {n / wave:.2f} waves of {wave}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", [9, 191, 257])
def test_an_unaligned_view_gives_the_bits_of_its_copy(dt, c):
    torch = _torch()
    from simple_tip_b200.core.deepgini import DeepGini
    from simple_tip_b200.core.quantifiers import MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy

    p_dev = torch.from_numpy(np.concatenate([_crafted(c, dt, seed=c), _rows(300, c, dt, seed=c)])).cuda()
    view = p_dev[1:]
    assert view.data_ptr() % 16 != 0 and view.is_contiguous()
    copy = view.clone()
    for cls in (DeepGini, MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy):
        a, b = cls.calculate(view), cls.calculate(copy)
        assert np.array_equal(a[0], b[0]) and _diff_rows(a[1], b[1]).size == 0, (cls.__name__, _route(c, dt))


# ---------------------------------------------------------------------------------------------------------------
# c. Non-finite rows
# ---------------------------------------------------------------------------------------------------------------
def _nan_rows(c, dt, seed):
    rng = np.random.default_rng(seed)
    rows = []

    def row(nan=(), inf=()):
        r = rng.uniform(0, 0.1, size=c)
        r[c // 4] = 0.9                                   # a clear finite maximum the NaN must beat
        r[list(inf)] = np.inf
        r[list(nan)] = np.nan
        rows.append(r)

    row(nan=[0])
    row(nan=[c // 2])
    row(nan=[c - 1])
    row(nan=[33, 31])                                     # two NaNs, the first in the higher lane
    row(nan=[c - 1, 2])
    row(nan=[39, 7])                                      # two NaNs in the same lane
    row(nan=[c - 1], inf=[1])
    row(nan=[1], inf=[0])
    row(nan=[c // 2], inf=[c // 4 + 1, c - 2])
    row(nan=list(range(c)))                               # all NaN
    row(nan=list(range(5, c, 3)))
    row()                                                 # finite rows beside them
    row(inf=[c - 1])
    return np.array(rows, dtype=dt)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", [40, 300])
def test_nan_rows_follow_numpy(dt, c):
    torch = _torch()
    from simple_tip_b200.core.deepgini import DeepGini
    from simple_tip_b200.core.quantifiers import MaxSoftmax, PredictionConfidenceScore, SoftmaxEntropy

    p = _nan_rows(c, dt, seed=c)
    p = np.concatenate([p, _rows(40, c, dt, seed=c), p])    # the NaN rows in two different blocks
    p_dev = torch.from_numpy(p).cuda()
    want_pred = np.argmax(p, axis=1)
    failed = []
    for cls, oracle in ((DeepGini, np_oracle.deepgini_oracle), (MaxSoftmax, QO.max_softmax),
                        (PredictionConfidenceScore, QO.pcs), (SoftmaxEntropy, QO.softmax_entropy)):
        pred, val = cls.calculate(p_dev)
        if not np.array_equal(pred, want_pred):
            failed.append((cls.__name__, "pred", np.flatnonzero(pred != want_pred)[:8].tolist()))
        want = oracle(p)[1]
        if cls is SoftmaxEntropy:                          # NumPy's sum of the kernel's own terms (libm's log2 aside)
            want = -np.sum(_terms(p_dev), axis=1)
            assert np.array_equal(np.isnan(want), np.isnan(oracle(p)[1]))
        if not np.array_equal(val, want, equal_nan=True) or _diff_rows(val, want).size:
            failed.append((cls.__name__, "value", _diff_rows(val, want)[:8].tolist()))
    print(f"\nc = {c} {np.dtype(dt).name} ({_route(c, dt)}): {int(np.isnan(p).any(axis=1).sum())} rows with NaN")
    assert not failed, failed


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", [12, 32, 33, 100])
def test_nan_samples_vote_for_their_numpy_argmax(dt, c):
    from simple_tip_b200.core.quantifiers import VariationRatio

    rng = np.random.default_rng(c)
    n, s = 50, 20
    p = rng.integers(0, 4, size=(n, s, c)).astype(dt) / 4
    hit = rng.random((n, s)) < 0.3
    cols = rng.integers(0, c, size=(n, s))
    p[hit, cols[hit]] = np.nan
    p[:, 0, 0] = np.nan                                   # column 0
    p[:, 1, c - 1] = np.nan                               # the last column
    p[:, 2, [min(31, c - 1), min(33, c - 1)]] = np.nan    # two NaNs, the first in the higher lane
    p[:5] = np.nan                                        # every sample all NaN: votes for class 0
    pred, vr = VariationRatio.calculate(p)
    wp, wv = QO.variation_ratio(p)
    print(f"\nc = {c} {np.dtype(dt).name}: {int(np.isnan(p).any(axis=2).sum())} of {n * s} samples hold a NaN")
    assert np.array_equal(pred, wp) and np.array_equal(vr, wv), (np.flatnonzero(pred != wp)[:8],
                                                                 np.flatnonzero(vr != wv)[:8])


# ---------------------------------------------------------------------------------------------------------------
# d. Votes at their edges
# ---------------------------------------------------------------------------------------------------------------
VOTE_CASES = [  # (S, c, rows per block, argmax, counts)
    (1, 32, 256, "thread", "shared"), (1, 33, 256, "warp", "shared"),
    (256, 32, 1, "thread", "shared"), (257, 33, 1, "warp", "shared"), (600, 32, 1, "thread", "shared"),
    (600, 33, 1, "warp", "shared"),
    (1, 47, 256, "warp", "shared"),          # 12032: under
    (1, 48, 256, "warp", "shared"),          # 12288: exactly at
    (1, 49, 250, "warp", "shared"),          # 12250: under, rows_per_block set by the width
    (2, 96, 128, "warp", "shared"),          # 12288: at
    (3, 97, 85, "warp", "shared"),           # 8245
    (257, 12287, 1, "warp", "shared"),       # one row, just under
    (1, 12288, 1, "warp", "shared"),         # one row, exactly at
    (1, 12289, 1, "warp", "global"),         # one row, just over
    (600, 12289, 1, "warp", "global"),
]


def _vote_probs(n, s, c, dt, seed):
    """Quarter-step values: many tied maxima inside a sample, and few distinct votes, so the mode ties too."""
    rng = np.random.default_rng(seed)
    p = rng.integers(0, 4, size=(n, s, c)).astype(dt) / 4
    top = rng.integers(0, min(c, 3), size=(n, s))
    np.put_along_axis(p, top[..., None], 1.0, axis=2)
    p[:, ::3, c - 1] = 1.0                                 # a tie of the maximum with the last class
    return p


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("s,c,rpb,argmax,counts", VOTE_CASES)
def test_votes_at_their_edges(dt, s, c, rpb, argmax, counts):
    torch = _torch()
    from simple_tip_b200.core.quantifiers import Votes

    assert _vote_route(s, c) == (rpb, argmax, counts)
    n = min(3 * rpb + 1, max(3, 4_000_000 // (s * c)))
    assert n % rpb != 0 or rpb == 1
    p = _vote_probs(n, s, c, dt, seed=s * c)
    votes = Votes(n, c, "cuda")
    votes.add(torch.from_numpy(p).cuda(), s, sample_stride=c, row_stride=s * c)
    want_counts = QO.vote_counts(p)
    assert np.array_equal(votes.counts.cpu().numpy(), want_counts)
    pred, vr = votes.finish(s)
    wp, wv = QO.variation_ratio(p)
    assert np.array_equal(pred, wp) and np.array_equal(vr, wv)
    print(f"\nS = {s}, c = {c} {np.dtype(dt).name}: {n} rows, {rpb} per block, {argmax} argmax, {counts} counts, "
          f"{int((want_counts == want_counts.max(axis=1, keepdims=True)).sum(axis=1).max())} classes tied at most")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("s,c", [(5, 7), (3, 40), (300, 33)])
def test_votes_read_a_padded_buffer_through_both_strides(dt, s, c):
    """Sample s of row i at i * row_stride + s * sample_stride, with gaps between samples and between rows; the gaps
    hold values that would win every vote if they were read."""
    torch = _torch()
    from simple_tip_b200.core.quantifiers import Votes

    n = 37
    p = _vote_probs(n, s, c, dt, seed=s + c)
    buf = np.full((n, s + 2, c + 3), 2.0, dtype=dt)
    buf[:, :, c:] = np.nan
    buf[:, :s, :c] = p
    votes = Votes(n, c, "cuda")
    votes.add(torch.from_numpy(buf).cuda(), s, sample_stride=c + 3, row_stride=(s + 2) * (c + 3))
    assert np.array_equal(votes.counts.cpu().numpy(), QO.vote_counts(p))
    pred, vr = votes.finish(s)
    wp, wv = QO.variation_ratio(p)
    assert np.array_equal(pred, wp) and np.array_equal(vr, wv)
