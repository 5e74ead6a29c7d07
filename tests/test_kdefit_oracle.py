"""CPU tests of LSA's device-fit reference and host side: the np.var chains of oracle/kdefit_oracle.py pinned to the
installed NumPy, its float64 fit pinned to StableGaussianKDE's host fit, the comparisons rejecting injected defects,
backend selection, and the errors raised before any launch."""
import numpy as np
import pytest

from oracle import kdefit_oracle as K
from simple_tip_b200 import _lib
from simple_tip_b200.core import surprise
from simple_tip_b200.core.stable_kde import StableGaussianKDE


def _traces(n, d, dtype, seed=0):
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.normal(size=(n, d)) * rng.uniform(0.1, 3, d) + rng.normal(size=d), 0)
    x[:, 0] = 0.0
    if d > 1:
        x[:, 1] = 1e4 + rng.normal(size=n)          # a large offset: reordering or fusing shows in the last bits
    if d > 2:
        x[:, 2] = 3.7
    return np.ascontiguousarray(x.astype(dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,d", [(1, 1), (2, 1), (7, 1), (3000, 1), (1, 5), (7, 3), (3000, 40), (20000, 6)])
def test_var_chains_are_np_var_bit_for_bit(n, d, dtype):
    x = _traces(n, d, dtype, seed=n + d)
    assert np.array_equal(K.var(x), np.var(x, axis=0))
    if d == 1:
        xo = np.ascontiguousarray(x + dtype(1e4))
        assert np.array_equal(K.var(xo), np.var(xo, axis=0))


def test_var_comparison_rejects_injected_defects():
    x = _traces(3000, 6, np.float32, seed=4)
    want = np.var(x, axis=0)
    assert not np.array_equal(K.var(x, fma=True), want)                 # an FMA'd square
    assert not np.array_equal(K.var(x[1:]), want)                        # a dropped row
    assert not np.array_equal(K.var(x[:, [0, 1, 3, 3, 4, 5]]), want)     # a wrong column


def _host_kde(x):
    """StableGaussianKDE's host fit (stable_kde.py:20-77) without the device upload."""
    kde = StableGaussianKDE.__new__(StableGaussianKDE)
    kde.dataset = np.atleast_2d(x.T).astype(np.float64)
    kde.d, kde.n = kde.dataset.shape
    kde.weights = np.ones(kde.n) / kde.n
    kde.neff = 1.0 / np.sum(kde.weights ** 2)
    kde._compute_covariance()
    return kde


def _cond_data(n, d, spread, seed=3):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(d, d)))
    return (rng.normal(size=(n, d)) * np.geomspace(1, spread, d)) @ q.T + 2.0


@pytest.mark.parametrize("spread", [3.0, 1e3])
def test_oracle_fit_is_the_host_fit(spread):
    x = _cond_data(3000, 12, spread)
    kde, ref = _host_kde(x), K.fit(x)
    assert ref["factor"] == kde.factor and ref["rounds"] == 1 and not kde.prepare_failed
    np.testing.assert_allclose(ref["covariance"], kde._data_covariance, rtol=1e-11,
                               atol=1e-13 * np.abs(kde._data_covariance).max())
    w = np.linalg.cholesky(kde.inv_cov)
    np.testing.assert_allclose(ref["whitening"], w, rtol=1e-8, atol=1e-10 * np.abs(w).max())
    assert abs(ref["log_det"] - kde.log_det) <= 1e-9 * abs(kde.log_det)
    assert abs(ref["norm_factor"] - kde._norm_factor) <= 1e-9 * kde._norm_factor
    p = (kde.dataset.T - kde.dataset.mean(axis=1)) @ w
    np.testing.assert_allclose(ref["p"], p, rtol=1e-8, atol=1e-10 * np.abs(p).max())


@pytest.mark.parametrize("kind", ["constant", "duplicated", "all_zero"])
def test_oracle_fit_takes_the_host_branches(kind):
    x = np.random.default_rng(1).normal(size=(400, 6))
    if kind == "constant":
        x[:, 4] = 2.5
    elif kind == "duplicated":
        x[:, 5] = x[:, 0]
    else:
        x = np.zeros((50, 6))
    kde, ref = _host_kde(x), K.fit(x)
    assert ref["prepare_failed"] == kde.prepare_failed == (kind != "all_zero")


def test_bounds_hold_for_the_host_fit_and_reject_defects():
    x = _cond_data(4000, 10, 30.0)
    ref = K.fit(x)
    b = K.cov_bound(x)
    host = np.atleast_2d(np.cov(x.T, rowvar=1, bias=False, aweights=np.ones(4000) / 4000))
    assert np.all(np.abs(host - ref["covariance"]) <= b)
    dropped = np.cov(x[1:].T, rowvar=1, bias=False, aweights=np.ones(3999) / 3999)
    assert np.any(np.abs(dropped - ref["covariance"]) > b)
    swapped = host[np.ix_([1, 0] + list(range(2, 10)), [1, 0] + list(range(2, 10)))]
    assert np.any(np.abs(swapped - ref["covariance"]) > b)
    w = np.linalg.cholesky(np.linalg.inv(host * ref["factor"] ** 2))
    w_b = K.whitening_bound(ref, b)
    assert np.linalg.norm(w - ref["whitening"]) <= w_b
    p = ((x - x.mean(axis=0)) @ w).astype(np.float32)
    assert np.all(np.abs(p - ref["p"]) <= K.p_bound(x, None, ref, w_b))
    assert np.any(np.abs(p[:, ::-1] - ref["p"]) > K.p_bound(x, None, ref, w_b))


def test_host_backend_stays_the_default(monkeypatch):
    monkeypatch.delenv("B200TIP_KDE", raising=False)
    assert surprise._kde_backend(None) == "host"
    monkeypatch.setenv("B200TIP_KDE", "device")
    assert surprise._kde_backend(None) == "device"
    assert surprise._kde_backend("host") == "host"


def test_unknown_backend_is_rejected(monkeypatch):
    x = _traces(60, 4, np.float32)
    with pytest.raises(ValueError, match="backend"):
        surprise.LSA(x, backend="cpu")
    monkeypatch.setenv("B200TIP_KDE", "cuda")
    with pytest.raises(ValueError, match="backend"):
        surprise.LSA(x)


def test_device_backend_errors_before_any_launch(monkeypatch):
    import torch

    class TwoRanks:
        world = 2

    with pytest.raises(NotImplementedError, match="not sharded"):
        surprise.LSA(_traces(60, 4, np.float32), backend="device", comm=TwoRanks())
    with pytest.raises(ValueError, match="`dataset` input should have multiple elements"):
        StableGaussianKDE.from_device(np.zeros((1, 1), dtype=np.float32))
    if torch.cuda.is_available():
        return
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        surprise.LSA(_traces(60, 4, np.float32), backend="device")
    monkeypatch.setenv("B200TIP_KDE", "device")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        surprise.MultiModalSA.build_by_class(_traces(60, 4, np.float32), np.arange(60) % 2,
                                             lambda x, y: surprise.LSA(x))


def test_new_entry_points_are_declared_and_bound():
    for name in ("tip_col_var", "tip_whiten_dmma"):
        assert name in set(_lib.symbols())
        assert hasattr(_lib.load(), name)
