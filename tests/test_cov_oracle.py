"""CPU: the float64 restatement of EmpiricalCovariance().fit (oracle/cov_oracle.py) pinned to NumPy, scipy and
sklearn, and the comparisons the GPU tests use shown to reject injected defects."""
import warnings

import numpy as np
import pytest
from scipy import linalg

from oracle import cov_oracle as C


def _data(n, d, dtype, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(n, d)) * rng.uniform(0.1, 30, size=d) + rng.normal(size=d) * 5).astype(dtype)


def _scipy(x):
    d = x.shape[1]
    cov = np.cov(x.T, bias=1).reshape(d, d)
    p, rank = linalg.pinvh(cov, return_rank=True)
    s = linalg.eigvalsh(cov)
    return cov, p, rank, s, C.cutoff(s, d)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,d", [(1, 1), (2, 1), (9, 1), (6000, 1), (1, 17), (2, 17), (1000, 17), (6000, 300),
                                 (2000, 2304)])
def test_location_is_numpys_mean_bit_for_bit(n, d, dtype):
    x = _data(n, d, dtype, seed=n + d)
    loc = C.location(x)
    assert loc.dtype == x.dtype and np.array_equal(loc, x.mean(0))
    # np.cov's centring mean: the float64 copy of x.T, averaged along its rows
    assert np.array_equal(C.mean64(x), np.array(x.T, ndmin=2, dtype=np.float64).mean(axis=1))


def test_location_matches_sklearn_and_rejects_a_float64_accumulation(monkeypatch):
    from sklearn.covariance import EmpiricalCovariance

    x = _data(6000, 64, np.float32, seed=3)
    assert np.array_equal(C.location(x), EmpiricalCovariance().fit(x).location_)
    # defect: the float32 location accumulated in float64
    monkeypatch.setattr(C, "_column_sums", lambda a, acc: np.sum(a.astype(np.float64), axis=0).astype(acc))
    assert not np.array_equal(C.location(x), x.mean(0))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_covariance_within_the_scatter_bound_of_np_cov(dtype):
    x = _data(3000, 40, dtype, seed=4)
    ref = C.fit(x)
    cov = np.cov(x.T, bias=1)
    b = C.scatter_bound(x)
    assert np.all(np.abs(ref["covariance"] - cov) <= b)
    scale = np.sqrt(np.outer(np.diag(cov), np.diag(cov)))
    assert float(np.max(b / scale)) < 1e-9                 # the bound is not vacuous


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("kind", C.RANK_CASES)
def test_rank_and_precision_match_scipy_on_gap_spectra(kind, dtype):
    x = C.rank_case(kind, seed=1, dtype=dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cov, p, rank, s, cut = _scipy(x)
    assert C.gap(s, cut) > C.RANK_GAP, "the spectrum has an eigenvalue near the cutoff"
    ref = C.fit(x)
    assert ref["rank"] == rank
    assert np.max(np.abs(ref["precision"] - p), initial=0.0) <= C.precision_bound(x, ref)
    if kind == "dead":
        assert ref["live"][0] == 12 and ref["live"].size == rank    # every live column adds one eigenvalue here
    if ref["live"].size:
        w = ref["w"]
        pl = ref["precision"][np.ix_(ref["live"], ref["live"])]
        assert np.max(np.abs(w @ w.T - pl)) <= C.precision_bound(x, ref)


def test_precision_and_scores_match_sklearn():
    from sklearn.covariance import EmpiricalCovariance

    x = _data(4000, 48, np.float64, seed=5)
    ref = C.fit(x)
    sk = EmpiricalCovariance().fit(x)
    assert np.max(np.abs(ref["precision"] - sk.precision_)) <= C.precision_bound(x, ref)
    test = _data(200, 48, np.float64, seed=6)
    np.testing.assert_allclose(C.scores(test, ref), sk.mahalanobis(test), rtol=1e-9)


def test_cutoff_with_n_instead_of_d_is_rejected(monkeypatch):
    x = C.rank_case("small_axis", seed=1)
    _, _, rank, s, cut = _scipy(x)
    assert C.gap(s, cut) > C.RANK_GAP and C.fit(x)["rank"] == rank == 2
    n = x.shape[0]
    monkeypatch.setattr(C, "cutoff", lambda s, d: float(n * C.EPS * np.max(np.abs(s))))
    assert C.fit(x)["rank"] != rank


def test_a_deflated_live_column_is_rejected():
    x = C.rank_case("dead", seed=1)
    _, p, rank, _, _ = _scipy(x)
    good = C.fit(x)
    assert good["rank"] == rank
    bad = C.fit(x, live=good["live"][1:])
    assert bad["rank"] != rank


def test_a_dropped_kept_eigenvalue_is_rejected(monkeypatch):
    x = C.rank_case("duplicated", seed=1)
    _, p, rank, _, _ = _scipy(x)
    good = C.fit(x)
    smallest = float(np.min(np.abs(good["eigenvalues"][good["keep"]])))
    monkeypatch.setattr(C, "cutoff", lambda s, d: smallest)
    bad = C.fit(x)
    assert bad["rank"] == rank - 1
    assert np.max(np.abs(bad["precision"] - p)) > C.precision_bound(x, good)


def test_score_bound_covers_the_fp32_whitening():
    x = _data(3000, 64, np.float32, seed=7)
    ref = C.fit(x)
    test = _data(300, 64, np.float32, seed=8)
    w32 = ref["w"].astype(np.float32)
    xc32 = (test[:, ref["live"]].astype(np.float64) - ref["location"][ref["live"]]).astype(np.float32)
    y = (xc32 @ w32).astype(np.float64)
    err = np.abs(np.sum(y * y, axis=1) - C.scores(test, ref))
    assert np.all(err <= C.score_bound(test, ref, C.precision_bound(x, ref)))
