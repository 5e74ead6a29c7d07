"""CPU: the float64 GaussianMixture reference (oracle/gmm_oracle.py) pinned to live sklearn started from the
reference's own initial state, after 1 and 2 iterations and at convergence."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.mixture import GaussianMixture

from oracle import gmm_oracle as G


def _blobs(seed, n=900, d=6, dead=0):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(3, d)) * 4.0
    lab = rng.integers(0, 3, size=n)
    x = centres[lab] + rng.normal(size=(n, d))
    if dead:
        x[:, :dead] = 0.0                 # dead ReLU units: constant columns, only reg_covar on their diagonal
    return x, lab


def _sklearn_from(init, k, max_iter, tol=1e-3, reg_covar=1e-6):
    w, mu, cov, _ = init
    return GaussianMixture(n_components=k, max_iter=max_iter, tol=tol, reg_covar=reg_covar, weights_init=w,
                           means_init=mu, precisions_init=np.linalg.inv(cov), init_params="random", random_state=0)


@pytest.mark.parametrize("dead", [0, 2])
@pytest.mark.parametrize("max_iter", [1, 2, 100])
def test_oracle_matches_live_sklearn(dead, max_iter):
    x, lab = _blobs(3 + dead, dead=dead)
    ref = G.fit(x, lab, 3, max_iter=max_iter)
    sk = _sklearn_from(ref["init"], 3, max_iter)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        sk.fit(x)
    assert sk.n_iter_ == ref["n_iter"] and sk.converged_ == ref["converged"]
    # sklearn starts from cholesky(inv(cov)) (a lower factor) where the reference uses inv(cholesky(cov))^T;
    # both give the same quadratic form up to rounding, amplified by cond(cov) <= 1e6 on the dead columns
    rtol = 1e-7 if dead else 1e-10
    np.testing.assert_allclose(ref["weights"], sk.weights_, rtol=rtol, atol=0)
    np.testing.assert_allclose(ref["means"], sk.means_, rtol=rtol, atol=1e-12)
    np.testing.assert_allclose(ref["covariances"], sk.covariances_, rtol=rtol, atol=1e-12)
    np.testing.assert_allclose(ref["prec_chol"], sk.precisions_cholesky_, rtol=rtol, atol=1e-9)
    assert abs(ref["lower_bound"] - sk.lower_bound_) <= 1e-10 * abs(sk.lower_bound_)
    np.testing.assert_allclose(ref["lower_bounds"], sk.lower_bounds_, rtol=1e-10)
    np.testing.assert_allclose(G.score_samples(x, ref["weights"], ref["means"], ref["prec_chol"]), sk.score_samples(x),
                               rtol=1e-9)


def test_oracle_records_change_and_margin():
    x, lab = _blobs(11)
    ref = G.fit(x, lab, 3, max_iter=100, tol=1e-3)
    assert ref["converged"] and len(ref["changes"]) == ref["n_iter"] == len(ref["margins"])
    assert ref["changes"][0] == np.inf
    for i, (c, m) in enumerate(zip(ref["changes"], ref["margins"])):
        assert m == abs(abs(c) - 1e-3)
        assert (abs(c) < 1e-3) == (i == ref["n_iter"] - 1)


def test_oracle_init_is_sklearns_initialize_from_one_hot_labels():
    x, lab = _blobs(5, n=300)
    w, mu, cov, prec = G.initialize(x, lab, 3, 1e-6)
    sk = GaussianMixture(n_components=3, reg_covar=1e-6)
    resp = np.zeros((x.shape[0], 3))
    resp[np.arange(x.shape[0]), lab] = 1.0
    sk._initialize(x, resp)
    np.testing.assert_array_equal(w, sk.weights_)
    np.testing.assert_allclose(mu, sk.means_, rtol=1e-14)
    np.testing.assert_allclose(cov, sk.covariances_, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(prec, sk.precisions_cholesky_, rtol=1e-10, atol=1e-12)


def test_non_positive_definite_covariance_raises():
    cov = np.array([[[1.0, 2.0], [2.0, 1.0]]])
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        G.precision_cholesky(cov)
