"""Float64 NumPy reference of sklearn's full-covariance GaussianMixture EM, started from given hard labels.

Restated from sklearn 1.9 (`sklearn/mixture/_gaussian_mixture.py`, `_base.py`):
- `initialize(x, labels, k, reg_covar)`: `_initialize` with one-hot responsibilities (weights = nk / n);
- `e_step`: `_estimate_log_gaussian_prob` ('full') + `_estimate_log_prob_resp` (scipy logsumexp) and the mean;
- `m_step`: `_estimate_gaussian_parameters` + `_compute_precision_cholesky`, weights normalised by their sum;
- `fit`: the `fit_predict` loop for n_init = 1 (change = bound - previous, previous = -inf first, stop when
  |change| < tol).  For every iteration it records the bound, the change and the change's margin to tol.

The quadratic forms are computed centred first, `|(x - mu) . L|^2`, as the device does; sklearn's
`X @ L - mu @ L` gives the same value up to rounding.  `error_bounds` is the fp64 error model of DESIGN.md §5b.
"""
from __future__ import annotations

import numpy as np
from scipy import linalg
from scipy.special import logsumexp

EPS = np.finfo(np.float64).eps
U = EPS / 2                       # unit roundoff of float64
LOG_2PI = np.log(2 * np.pi)


class FitError(ValueError):
    pass


def precision_cholesky(cov: np.ndarray) -> np.ndarray:
    """sklearn _compute_precision_cholesky ('full'): inv(cholesky(cov_k, lower))^T per component."""
    k, d, _ = cov.shape
    out = np.empty_like(cov)
    for j in range(k):
        try:
            c = linalg.cholesky(cov[j], lower=True)
        except linalg.LinAlgError:
            raise FitError("Fitting the mixture model failed because some components have ill-defined empirical "
                           "covariance")
        out[j] = linalg.solve_triangular(c, np.eye(d), lower=True).T
    return out


def log_det(prec_chol: np.ndarray) -> np.ndarray:
    return np.sum(np.log(np.diagonal(prec_chol, axis1=1, axis2=2)), axis=1)


def quad(x: np.ndarray, means: np.ndarray, prec_chol: np.ndarray) -> np.ndarray:
    """q[k, i] = |(x_i - mu_k) . L_k|^2, float64, upper triangle of L only."""
    x = np.asarray(x, dtype=np.float64)
    out = np.empty((means.shape[0], x.shape[0]))
    for j in range(means.shape[0]):
        y = (x - means[j]) @ np.triu(prec_chol[j])
        out[j] = np.sum(y * y, axis=1)
    return out


def weighted_log_prob(q: np.ndarray, d: int, weights: np.ndarray, prec_chol: np.ndarray) -> np.ndarray:
    """[n, k]: (-.5 (d log 2pi + q) + log det) + log w."""
    return (-0.5 * (d * LOG_2PI + q.T) + log_det(prec_chol)) + np.log(weights)


def e_step(x, weights, means, prec_chol):
    """(mean of log_prob_norm, log_prob_norm [n], resp [n, k])."""
    q = quad(x, means, prec_chol)
    wlp = weighted_log_prob(q, x.shape[1], weights, prec_chol)
    lpn = logsumexp(wlp, axis=1)
    return float(np.mean(lpn)), lpn, np.exp(wlp - lpn[:, None])


def moments(x, resp):
    """(nk, resp^T x, means) as sklearn _estimate_gaussian_parameters."""
    x = np.asarray(x, dtype=np.float64)
    nk = resp.sum(axis=0) + 10 * EPS
    sums = resp.T @ x
    return nk, sums, sums / nk[:, None]


def scatter(x, resp, means):
    """Unnormalised S_k = sum_i r_ik (x_i - mu_k)(x_i - mu_k)^T, [k, d, d]."""
    x = np.asarray(x, dtype=np.float64)
    out = np.empty((means.shape[0], x.shape[1], x.shape[1]))
    for j in range(means.shape[0]):
        diff = x - means[j]
        out[j] = (resp[:, j] * diff.T) @ diff
    return out


def m_params(x, resp, reg_covar):
    """(nk, means, covariances) of _estimate_gaussian_parameters."""
    nk, _, means = moments(x, resp)
    cov = scatter(x, resp, means) / nk[:, None, None]
    cov += reg_covar * np.eye(x.shape[1])[None]
    return nk, means, cov


def m_step(x, resp, reg_covar):
    """(weights, means, covariances, prec_chol) after sklearn's _m_step."""
    nk, means, cov = m_params(x, resp, reg_covar)
    return nk / nk.sum(), means, cov, precision_cholesky(cov)


def initialize(x, labels, k, reg_covar):
    """sklearn _initialize from hard labels: (weights, means, covariances, prec_chol)."""
    resp = np.zeros((x.shape[0], k))
    resp[np.arange(x.shape[0]), np.asarray(labels)] = 1.0
    nk, means, cov = m_params(x, resp, reg_covar)
    return nk / x.shape[0], means, cov, precision_cholesky(cov)


def em_step(x, weights, means, prec_chol, reg_covar):
    """One EM iteration: (bound of the E-step, weights, means, covariances, prec_chol)."""
    lb, _, resp = e_step(x, weights, means, prec_chol)
    return (lb,) + m_step(x, resp, reg_covar)


def fit(x, labels, k, max_iter=100, tol=1e-3, reg_covar=1e-6):
    """sklearn fit_predict (n_init = 1) from hard initial labels.  Returns a dict: init (the initial state), the
    final weights / means / covariances / prec_chol, n_iter, converged, lower_bound, lower_bounds, and per
    iteration `changes` and `margins` (| |change| - tol |: how far the stop decision is from flipping)."""
    x = np.asarray(x, dtype=np.float64)
    state = initialize(x, labels, k, reg_covar)
    init = state
    lower_bound, bounds, changes, margins, converged, n_iter = -np.inf, [], [], [], False, 0
    for n_iter in range(1, max_iter + 1):
        prev = lower_bound
        lower_bound, *state = em_step(x, state[0], state[1], state[3], reg_covar)
        change = lower_bound - prev
        bounds.append(lower_bound)
        changes.append(change)
        margins.append(abs(abs(change) - tol))
        if abs(change) < tol:
            converged = True
            break
    w, mu, cov, prec = state
    return {"init": init, "weights": w, "means": mu, "covariances": cov, "prec_chol": prec, "n_iter": n_iter,
            "converged": converged, "lower_bound": lower_bound, "lower_bounds": bounds, "changes": changes,
            "margins": margins}


def score_samples(x, weights, means, prec_chol):
    return e_step(np.asarray(x, dtype=np.float64), weights, means, prec_chol)[1]


# ---- fp64 error model (DESIGN.md §5b) ---------------------------------------------------------------------------
def gamma(m: int) -> float:
    """Higham's gamma_m = m u / (1 - m u): the relative bound of an m-term float64 dot product / sum."""
    return m * U / (1 - m * U)


def quad_bound(x, means, prec_chol) -> np.ndarray:
    """|q_device - q_exact| <= this, per (k, i): centring (1 rounding per element), the dot product of length
    <= d per output column (gamma_d relative to sum |x - mu| |L|), the square (2 u) and the row sum of d squares
    (gamma_d relative to the sum of the squares)."""
    x = np.asarray(x, dtype=np.float64)
    d = x.shape[1]
    out = np.empty((means.shape[0], x.shape[0]))
    for j in range(means.shape[0]):
        a = np.abs(x - means[j])
        yabs = a @ np.abs(np.triu(prec_chol[j]))
        y = (x - means[j]) @ np.triu(prec_chol[j])
        e_y = gamma(d + 1) * yabs
        out[j] = np.sum(2 * np.abs(y) * e_y + e_y * e_y, axis=1) + gamma(d + 2) * np.sum(y * y, axis=1)
    return out
