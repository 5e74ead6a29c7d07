"""Float64 NumPy restatement of LSA's fit (the variance-ranked column selection and `StableGaussianKDE`'s fit), and
the error bounds the device fit is held to (DESIGN.md §5d).

- `var(x)`: NumPy 2.3's `np.var(x, axis=0)` as explicit chains: the input-dtype column sum (sequential over the
  rows for d >= 2, NumPy's pairwise sum for d == 1), divided by n in double and rounded once; `x - mean` in x's
  dtype; the square as its own rounding; the same reduce and division.  `fma=True` fuses the square into the sum
  (a defect the comparison must reject).
- `fit(x, cols)`: StableGaussianKDE(x[:, cols].T)'s fit in float64: Scott factor, np.cov(bias=False, aweights=1/n)
  written out, the stabilisation loop (the diagonal REPLACED by 1e-10 * 2^k while an eigenvalue of cov * f^2 is
  <= 0, failing past 1e-5), inv, cholesky(2 pi covariance), W = cholesky(inv_cov) and p = (x[:, cols] - mean) @ W.
- `cov_bound`: entrywise |device covariance - reference covariance|, cov_oracle.scatter_bound adapted to the weights
  1/n, the factor 1/fact and np.cov's weighted mean.
- `whitening_bound`: ||W_device - W_reference||_F, first order in the covariance error eps_C (normwise, relative):
  W = R^-T for the reversed Cholesky factor R of C (C = R R^T), so kappa^1.5 eps_C; plus kappa^2 c d u for the
  inverse and the factorisations.  `residual_bound`: ||C_ref f^2 W W^T - I||_2, first order in kappa (eps_C +
  d^2 u) and no more than 8x the reference's own residual beyond that; it stays informative at large kappa.
- `p_bound`: entrywise |p_device - p_reference|, with the fp32 rounding of the device operand.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.cov_oracle import U, U32, _pairwise, gamma

MAX_INCREMENT = 1e-5


def _reduce_rows(a: np.ndarray, t, fused_with: np.ndarray = None) -> np.ndarray:
    """np.add.reduce(a, axis=0) in dtype t: sequential over the rows for d >= 2, pairwise for d == 1.
    fused_with: a FUSED multiply-add chain s = fl(s + e * e) over its rows instead (float32 only)."""
    if fused_with is not None:
        s = np.zeros(fused_with.shape[1], dtype=t)
        for e in fused_with:
            s = (s.astype(np.float64) + e.astype(np.float64) * e.astype(np.float64)).astype(t)
        return s
    if a.shape[1] == 1:
        return np.array([t(t(0.0) + _pairwise(np.ascontiguousarray(a[:, 0]), t))], dtype=t)
    s = np.zeros(a.shape[1], dtype=t)
    for row in a:
        s = s + row                   # one IEEE add per element, in row order
    return s


def var(x: np.ndarray, fma: bool = False) -> np.ndarray:
    """np.var(x, axis=0) of a C-contiguous [n, d] float32 / float64 matrix, restated as explicit chains."""
    t = x.dtype.type
    n = x.shape[0]
    mean = (_reduce_rows(x, t).astype(np.float64) / n).astype(x.dtype)
    e = x - mean                      # arr - arrmean, in x's dtype
    s2 = _reduce_rows(None, t, fused_with=e) if fma else _reduce_rows(e * e, t)
    return (s2.astype(np.float64) / n).astype(x.dtype)


def fit(x: np.ndarray, cols: np.ndarray = None) -> dict:
    """StableGaussianKDE(x[:, cols].T)'s fit in float64 (x: [n, D]).  Returns the stabilised data covariance
    (unscaled), its inverse, factor, whitening W, the column mean, p, log_det, norm_factor, norm, log_norm, rounds
    and prepare_failed (the later entries missing when the fit failed)."""
    data = (x if cols is None else x[:, cols]).astype(np.float64)
    n, d = data.shape
    w = np.ones(n) / n
    factor = float(np.power(1.0 / np.sum(w ** 2), -1.0 / (d + 4)))
    w_sum = w.sum()
    fact = w_sum - np.sum(w * w) / w_sum
    avg = (data * w[:, None]).sum(axis=0) / w_sum
    xc = data - avg
    cov = (xc.T @ (xc * w[:, None])) * (1.0 / fact)
    out = {"factor": factor, "fact": fact, "mean": data.mean(axis=0)}
    increment, rounds = 1e-10, 0
    while True:
        rounds += 1
        if not np.any(np.linalg.eigh(cov * factor ** 2)[0] <= 0):
            break
        np.fill_diagonal(cov, increment)
        if increment > MAX_INCREMENT:
            out.update(rounds=rounds, prepare_failed=True)
            return out
        increment += increment
    inv = np.linalg.inv(cov)
    covariance = cov * factor ** 2
    inv_cov = inv / factor ** 2
    wl = np.linalg.cholesky(inv_cov)
    diag = np.diag(wl)
    norm = math.pow(2 * math.pi, -d / 2.0)
    for i in range(d):
        norm *= diag[i]
    out.update(rounds=rounds, prepare_failed=False, covariance=cov, inv=inv, whitening=wl,
               log_det=float(2 * np.log(np.diag(np.linalg.cholesky(covariance * 2 * np.pi))).sum()),
               norm_factor=float(np.sqrt(np.linalg.det(2 * np.pi * covariance))), norm=norm,
               log_norm=-d / 2.0 * math.log(2 * math.pi) + float(np.sum(np.log(diag))),
               p=(data - out["mean"]) @ wl)
    return out


def cov_bound(x: np.ndarray, cols: np.ndarray = None) -> np.ndarray:
    """Entrywise bound on |device covariance - fit(x, cols)['covariance']| (before any stabilisation).  Each side:
    its centring mean's error delta (a weighted sum of n terms and a division), the weight, centring and product
    roundings, an (n + 3)-term float64 accumulation over |x_a - m_a| + delta_a, the exact effect of centring on a
    perturbed mean (delta_a delta_b), and the reciprocal of fact and its product; doubled for the two sides."""
    data = (x if cols is None else x[:, cols]).astype(np.float64)
    n = data.shape[0]
    w_sum = (np.ones(n) / n).sum()
    fact = w_sum - n * (1.0 / n) ** 2 / w_sum
    m = data.mean(axis=0)
    delta = gamma(n + 2) * np.abs(data).sum(axis=0) / n + U * np.abs(m)
    a = np.abs(data - m) + delta
    cov = ((data - m).T @ (data - m)) / n / fact
    return 2.0 * (gamma(n + 3) * (a.T @ a) / n + np.outer(delta, delta)) / fact + 4 * U * np.abs(cov)


def kappa(cov: np.ndarray) -> float:
    s = np.linalg.eigvalsh(cov)
    return float(s.max() / s.min())


def _eps_c(cov: np.ndarray, cov_b: np.ndarray) -> float:
    return float(np.linalg.norm(cov_b, "fro") / np.linalg.eigvalsh(cov).max())


def whitening_bound(ref: dict, cov_b: np.ndarray) -> float:
    """Bound on ||W_device - ref['whitening']||_F (cov_b: cov_bound of the same rows)."""
    d = ref["covariance"].shape[0]
    k = kappa(ref["covariance"])
    rel = k ** 1.5 * _eps_c(ref["covariance"], cov_b) + k ** 2 * 16 * d * U
    return 2.0 * rel * float(np.linalg.norm(ref["whitening"], 2))


def host_residual(ref: dict) -> float:
    """||C f^2 W W^T - I||_2 of the reference's own W (LAPACK's inverse and Cholesky on the same matrix)."""
    c, w = ref["covariance"] * ref["factor"] ** 2, ref["whitening"]
    return float(np.linalg.norm(c @ (w @ w.T) - np.eye(c.shape[0]), 2))


def residual_bound(ref: dict, cov_b: np.ndarray) -> float:
    """Bound on ||ref['covariance'] f^2 W W^T - I||_2 for the device's W: the covariance error through the inverse
    (2 kappa eps_C), the inverse's and the Cholesky factor's rounding (8 d^2 u kappa: an LU inverse's residual and
    the factor's backward error, each d u kappa times a norm conversion of d), and 8x the reference's own residual,
    which measures how these factorisations behave on this matrix."""
    d = ref["covariance"].shape[0]
    k = kappa(ref["covariance"])
    return 2.0 * k * _eps_c(ref["covariance"], cov_b) + 8 * d * d * U * k + 8 * host_residual(ref)


def p_bound(x: np.ndarray, cols: np.ndarray, ref: dict, w_b: float) -> np.ndarray:
    """Entrywise bound on |p_device - ref['p']|: the whitening's error (w_b, normwise) over the centred rows, the
    centring mean's error, a (d + 1)-term float64 accumulation on each side, and the fp32 rounding of p_device."""
    data = (x if cols is None else x[:, cols]).astype(np.float64)
    n, d = data.shape
    xc = np.abs(data - ref["mean"])
    aw = np.abs(ref["whitening"])
    delta = gamma(n + 1) * np.abs(data).sum(axis=0) / n
    body = xc.sum(axis=1, keepdims=True) * w_b + (delta @ aw)[None, :] + 2 * gamma(d + 1) * (xc @ aw)
    return body + 2 * U32 * (np.abs(ref["p"]) + body)
