"""CPU model of tip_nn_filter's acceptance window (DESIGN.md §4): for random and adversarial data the
row NumPy picks as nearest neighbour (np.linalg.norm in the input dtype + np.argmin, surprise.py:638-647)
always lies inside the window the kernel derives from ANY row's approximate distance — with the
tensor-core accumulation error pushed to its assumed worst case against us.  This checks the error
budget (measured bf16 rounding norms, fp32 centring, accumulation) independently of the hardware; the
GPU tests then check the kernel against the oracle bit for bit."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle.filter_oracle import _bf16  # noqa: E402
from oracle.filter_oracle import threshold_lo as _threshold  # noqa: E402

F32 = np.float32


def _check(x, Y, mu, rng):
    d = x.shape[0]
    xt, Yt = (x - mu).astype(F32), (Y - mu).astype(F32)           # fl32(x - mu), as pair_prep_kernel does
    xb, Yb = _bf16(xt), _bf16(Yt)
    errq = F32(np.sqrt(np.sum((xt.astype(np.float64) - xb) ** 2))) * F32(1.000001)
    errt = F32(np.sqrt(np.max(np.sum((Yt.astype(np.float64) - Yb) ** 2, axis=1)))) * F32(1.000001) * F32(1.000001)
    nx = F32(np.sum(xb.astype(np.float64) ** 2))
    rmax = F32(np.sqrt(np.max(np.sum(Yb.astype(np.float64) ** 2, axis=1)))) * F32(1.000001)
    r = F32(np.sqrt(nx) + rmax)
    e2 = F32(F32(2.0) * F32(errq + errt + F32(1.2e-7) * r) * F32(1.00001))
    k = ((d + 15) // 16) * 16 + 16
    g = F32(F32((k + 16) * 2.0 ** -23) * r * r)
    acc_exact = np.sum(Yb.astype(np.float64) ** 2, axis=1) - 2.0 * (Yb.astype(np.float64) @ xb.astype(np.float64))
    # the reference's arithmetic decides who the winner is
    dist_np = np.linalg.norm((x[None, None, :] - Y[None, :, :]).astype(F32), axis=2)[0]
    j_star = int(np.argmin(dist_np))
    ties = np.flatnonzero(dist_np == dist_np[j_star])            # every exactly tied row must be a candidate too
    worst = acc_exact + float(g)                                  # accumulation error against the winner
    for b in {int(np.argmin(acc_exact)), int(rng.integers(0, Y.shape[0])), j_star}:
        s = F32(max(F32(acc_exact[b] - float(g)) + nx, F32(0.0)))   # ... and in favour of the reference row
        thr = _threshold(s, nx, e2, g)
        if dist_np[b] >= dist_np[j_star]:                          # thr(b) must admit everything at least as near
            assert np.all(worst[ties] <= thr), (d, b, j_star, worst[ties], thr)


@pytest.mark.parametrize("d", [1, 9, 64, 128, 200, 1600])
def test_window_always_contains_numpys_argmin(d):
    rng = np.random.default_rng(d)
    for trial in range(12):
        n = int(rng.integers(2, 400))
        scale = float(rng.choice([1e-3, 1.0, 50.0]))
        offset = rng.normal(size=d).astype(F32) * F32(rng.choice([0.0, 5.0, 300.0]))
        Y = (rng.normal(size=(n, d)).astype(F32) * F32(scale) + offset).astype(F32)
        mu = Y.mean(axis=0, dtype=np.float64).astype(F32)
        kind = trial % 4
        if kind == 0:
            x = (rng.normal(size=d).astype(F32) * F32(scale) + offset).astype(F32)
        elif kind == 1:                                   # query equals a train row (distance 0) + a duplicate
            x = Y[0].copy()
            Y[-1] = Y[0]
        elif kind == 2:                                   # near ties: rows at almost the same distance
            x = (rng.normal(size=d).astype(F32) * F32(scale) + offset).astype(F32)
            base = Y[0] - x
            for i in range(1, min(n, 8)):
                Y[i] = (x + np.roll(base, i) * F32(1 + 1e-6 * i)).astype(F32)
        else:                                             # far-away query
            x = (offset + F32(40 * scale) * rng.normal(size=d).astype(F32)).astype(F32)
        _check(x, Y, mu, rng)


@pytest.mark.parametrize("d", [8, 24])
def test_window_is_tight_enough_for_aligned_rounding(d):
    """Adversarial construction: every coordinate of the query sits just below a bf16 rounding
    midpoint, the true nearest row just above it (so rounding moves them APART by ~|dx|+|dy|, all
    coordinates aligned), while a slightly farther row rounds onto the query (bf16 distance 0).
    The window must still keep the true winner — this is where the measured rounding norms are
    actually needed: a window built from a tenth of them loses the winner.  (Short traces only: from
    D ~ 100 on the accumulation budget g = (K+16) 2^-23 r^2 alone is as wide as the rounding term.)"""
    rng = np.random.default_rng(d)
    u = F32(2.0 ** -8)
    x = np.full(d, F32(1.0) + F32(0.98) * u, dtype=F32)            # rounds down to 1.0
    y_win = np.full(d, F32(1.0) + F32(1.02) * u, dtype=F32)        # rounds up to 1 + 2^-7; true gap 0.04 u
    y_near = x - F32(0.06) * u                                      # true gap 0.06 u, rounds onto bf16(x)
    far = (rng.normal(size=(20, d)).astype(F32) * F32(0.05) + F32(1.0)).astype(F32)   # same norm scale: small g
    Y = np.vstack([y_near[None, :], y_win[None, :], far]).astype(F32)
    mu = np.zeros(d, dtype=F32)
    assert np.array_equal(_bf16(x), _bf16(y_near)) and not np.array_equal(_bf16(x), _bf16(y_win))
    dist = np.linalg.norm((x[None, None, :] - Y[None, :, :]).astype(F32), axis=2)[0]
    assert int(np.argmin(dist)) == 1                                # NumPy's winner is the row that rounds away
    _check(x, Y, mu, rng)
    # teeth: the same data with a window built from a tenth of the rounding norms must lose the winner
    import tests.test_window_model as me

    orig = me._threshold
    try:
        me._threshold = lambda s, nx, e2, g: orig(s, nx, F32(e2 * F32(0.1)), g)
        with pytest.raises(AssertionError):
            me._check(x, Y, mu, rng)
    finally:
        me._threshold = orig


def _seed_s(ub, nx, q_err, t_rmax, t_err, gamma):
    """seed_row_min_bits() of csrc/common.cuh in float32."""
    r = F32(F32(np.sqrt(nx, dtype=F32)) + t_rmax)
    e = F32(F32(q_err + t_err + F32(1.2e-7) * r) * F32(1.00001))
    g = F32(gamma * r * r)
    d = F32(F32(ub * F32(1.000004)) + e)
    return F32(F32(d * d + g) * F32(1.000002))


@pytest.mark.parametrize("d", [3, 64, 128])
def test_seed_from_any_in_range_row_never_undercuts_that_rows_accumulator(d):
    """Stage-2 seeds (tip_nn_rerank next_seed_ub): the running minimum of a query starts at a value derived from
    its NumPy distance to SOME row of the range.  For the window proof that value must be >= the approximate squared
    distance the filter can compute for that row (worst-case accumulation error included): then every threshold
    derived from the seed is at least as wide as one the scan itself would reach, and the seed row is itself emitted."""
    rng = np.random.default_rng(100 + d)
    for trial in range(30):
        n = int(rng.integers(2, 200))
        scale = float(rng.choice([1e-3, 1.0, 50.0]))
        offset = rng.normal(size=d).astype(F32) * F32(rng.choice([0.0, 5.0, 300.0]))
        Y = (rng.normal(size=(n, d)).astype(F32) * F32(scale) + offset).astype(F32)
        x = Y[int(rng.integers(0, n))].copy() if trial % 3 == 0 else (rng.normal(size=d).astype(F32) * F32(scale) + offset).astype(F32)
        mu = Y.mean(axis=0, dtype=np.float64).astype(F32)
        xt, Yt = (x - mu).astype(F32), (Y - mu).astype(F32)
        xb, Yb = _bf16(xt), _bf16(Yt)
        errq = F32(np.sqrt(np.sum((xt.astype(np.float64) - xb) ** 2))) * F32(1.000001)
        errt = F32(np.sqrt(np.max(np.sum((Yt.astype(np.float64) - Yb) ** 2, axis=1)))) * F32(1.000001) * F32(1.000001)
        nx = F32(np.sum(xb.astype(np.float64) ** 2))
        rmax = F32(np.sqrt(np.max(np.sum(Yb.astype(np.float64) ** 2, axis=1)))) * F32(1.000001)
        k = ((d + 15) // 16) * 16 + 16
        gamma = F32((k + 16) * 2.0 ** -23)
        r = F32(np.sqrt(nx) + rmax)
        g = float(F32(gamma * r * r))
        dist_np = np.linalg.norm((x[None, None, :] - Y[None, :, :]).astype(F32), axis=2)[0]
        acc_exact = np.sum(Yb.astype(np.float64) ** 2, axis=1) - 2.0 * (Yb.astype(np.float64) @ xb.astype(np.float64))
        s_worst = acc_exact + g + float(nx)                      # the largest s the filter may compute for each row
        for j in rng.integers(0, n, size=5):
            seed = _seed_s(F32(dist_np[j]), nx, errq, rmax, errt, gamma)
            assert float(seed) >= s_worst[j], (d, trial, j, float(seed), s_worst[j])
            # and the threshold from the seed admits the seed row (it will be emitted as a candidate)
            e2 = F32(F32(2.0) * F32(errq + errt + F32(1.2e-7) * r) * F32(1.00001))
            assert acc_exact[j] + g <= _threshold(seed, nx, e2, F32(g))
