"""Float64 NumPy restatement of sklearn 1.9's `EmpiricalCovariance().fit` under the device's rules, and the error
bounds the device fit is held to (DESIGN.md §5c).

- `location(x)`: NumPy's `x.mean(0)`: a sequential sum over the rows in x's dtype for d >= 2, NumPy's pairwise sum
  for d == 1, then one division by n (done in double and rounded once);
- `mean64(x)`: the same sum in float64, np.cov's centring mean;
- `fit(x)`: covariance = centred scatter / n (float64); live columns = those whose centred values are not all
  exactly 0; the eigendecomposition of the live block; scipy pinvh's cutoff d * eps * max|s| with d counting every
  column; the precision (U / s) U^T over the kept eigenvalues; W = U diag(s^-1/2) over the kept s > 0.
- `scatter_bound(x)`: |device covariance - reference covariance| entrywise, both computed in float64;
- `precision_bound` / `score_bound`: the kept subspace, proportional to (scatter error + d u) * cond_kept;
- `gap(s, cutoff)`: how far the nearest eigenvalue lies from the cutoff, as a factor.  The device's rank must equal
  scipy's when every eigenvalue lies more than 100x above or below the cutoff.
"""
from __future__ import annotations

import numpy as np

EPS = np.finfo(np.float64).eps
U = EPS / 2                                   # unit roundoff of float64
U32 = np.finfo(np.float32).eps / 2            # unit roundoff of float32 (the scoring's whitening)
RANK_GAP = 100.0


def gamma(k, u=U) -> float:
    return k * u / (1 - k * u)


def _pairwise(a: np.ndarray, t) -> object:
    """NumPy's pairwise sum of the contiguous 1-D array a, accumulated in dtype t."""
    n = a.shape[0]
    if n < 8:
        r = t(0.0)
        for v in a:
            r = t(r + t(v))
        return r
    if n <= 128:
        r = [t(a[j]) for j in range(8)]
        lim = n - n % 8
        for i in range(8, lim, 8):
            for j in range(8):
                r[j] = t(r[j] + t(a[i + j]))
        res = t(t(t(r[0] + r[1]) + t(r[2] + r[3])) + t(t(r[4] + r[5]) + t(r[6] + r[7])))
        for i in range(lim, n):
            res = t(res + t(a[i]))
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return t(_pairwise(a[:n2], t) + _pairwise(a[n2:], t))


def _column_sums(x: np.ndarray, acc) -> np.ndarray:
    t = np.dtype(acc).type
    if x.shape[1] == 1:
        return np.array([t(t(0.0) + _pairwise(np.ascontiguousarray(x[:, 0]), t))], dtype=acc)
    s = np.zeros(x.shape[1], dtype=acc)
    for row in x:
        s = s + row.astype(acc)            # one IEEE add per element, in order
    return s


def location(x: np.ndarray) -> np.ndarray:
    """sklearn's location_ = x.mean(0), in x's dtype."""
    s = _column_sums(x, x.dtype)
    return (s.astype(np.float64) / x.shape[0]).astype(x.dtype)


def mean64(x: np.ndarray) -> np.ndarray:
    """np.cov(x.T)'s centring mean: the same sum in float64, / n."""
    return _column_sums(x, np.float64) / x.shape[0]


def cutoff(s: np.ndarray, d: int) -> float:
    """scipy pinvh: max(a.shape) * eps * max|s| (atol 0)."""
    return float(d * EPS * np.max(np.abs(s), initial=0.0))


def gap(s: np.ndarray, cut: float) -> float:
    """min over the eigenvalues of max(|s| / cut, cut / |s|) (inf when cut == 0 or every s == 0)."""
    a = np.abs(np.asarray(s, dtype=np.float64))
    if cut == 0.0:
        return np.inf
    with np.errstate(divide="ignore"):
        f = np.maximum(a / cut, cut / a)
    return float(np.min(f, initial=np.inf))


def fit(x: np.ndarray, live: np.ndarray = None) -> dict:
    """The device fit restated in float64 NumPy (x: [n, d], n >= 1).  live: the columns kept in the
    eigendecomposition (default: those whose centred values are not all exactly 0)."""
    n, d = x.shape
    x64 = x.astype(np.float64)
    m = mean64(x)
    xc = x64 - m
    cov = (xc.T @ xc) / n
    if live is None:
        live = np.flatnonzero(np.any(xc != 0.0, axis=0))
    precision = np.zeros((d, d))
    w = np.zeros((live.size, 0))
    s = np.zeros(0)
    cut, keep = 0.0, np.zeros(0, dtype=bool)
    if live.size:
        s, u = np.linalg.eigh(cov[np.ix_(live, live)])
        cut = cutoff(s, d)
        keep = np.abs(s) > cut
        uk, sk = u[:, keep], s[keep]
        precision[np.ix_(live, live)] = (uk * (1.0 / sk)) @ uk.T
        w = uk[:, sk > 0] / np.sqrt(sk[sk > 0])
    return {"location": location(x), "mean": m, "covariance": cov, "live": live, "eigenvalues": s, "cutoff": cut,
            "keep": keep, "rank": int(keep.sum()), "precision": precision, "w": w}


def scatter_bound(x: np.ndarray, cov: np.ndarray = None) -> np.ndarray:
    """Entrywise bound on |device covariance - fit(x)['covariance']|.  Each side: the mean's error delta (a sum of
    n terms, then a division), the centring and product roundings and an (n + 2)-term float64 accumulation over
    |x_a - m_a| + delta_a, plus the exact-arithmetic effect of centring on a perturbed mean (delta_a delta_b) and
    the final division; doubled because both sides are float64 computations of the same quantity."""
    n, _ = x.shape
    x64 = x.astype(np.float64)
    m = mean64(x)
    delta = gamma(n) * np.abs(x64).sum(axis=0) / n + U * np.abs(m)
    a = np.abs(x64 - m) + delta
    if cov is None:
        cov = ((x64 - m).T @ (x64 - m)) / n
    return 2.0 * (gamma(n + 2) * (a.T @ a) / n + np.outer(delta, delta) + U * np.abs(cov))


def _kept_spectrum(ref: dict):
    s = ref["eigenvalues"][ref["keep"]]
    return s, (float(np.max(np.abs(s))) / float(np.min(np.abs(s))) if s.size else 1.0)


def precision_bound(x: np.ndarray, ref: dict, cov_b: np.ndarray = None) -> float:
    """Entrywise bound on |device precision - reference precision| for a fit whose rank matches: the pseudo-inverse
    perturbation |dA+| <= mu |A+|^2 |dA| (mu < 2) with |dA| <= |cov_b|_F + 16 d u |A| (the scatter error, then
    both eigendecompositions' backward errors), i.e. 2 cond_kept (|cov_b|_F / s_max + 16 d u) / s_min."""
    s, cond = _kept_spectrum(ref)
    if not s.size:
        return 0.0
    d = x.shape[1]
    cov_b = scatter_bound(x, ref["covariance"]) if cov_b is None else cov_b
    live = ref["live"]
    eta = np.linalg.norm(cov_b[np.ix_(live, live)]) / np.max(np.abs(s)) + 16 * d * U
    return float(2.0 * cond * eta / np.min(np.abs(s)))


RANK_CASES = ("dead", "duplicated", "collinear", "n_lt_d", "one_row", "constant", "small_axis")


def rank_case(kind: str, seed: int = 0, dtype=np.float64) -> np.ndarray:
    """Rows whose covariance is singular in a known way (d >= 64 where the kind allows it):
    dead: ReLU rows with 8 all-zero and 4 constant columns; duplicated: 32 columns copied; collinear: 32 columns that
    are exact dyadic combinations of others (integer rows); n_lt_d: 40 rows of 256 columns; one_row: n = 1;
    constant: every row equal (dyadic values, so the mean is exact); small_axis: d = 2 with a second axis of
    variance 9e-14 (kept by d * eps * max, dropped by n * eps * max)."""
    rng = np.random.default_rng(seed)
    if kind == "small_axis":
        z = rng.normal(size=(1000, 2))
        z[:, 1] *= 3e-7
        return z.astype(dtype)
    n, d = {"n_lt_d": (40, 256), "one_row": (1, 64), "constant": (50, 64)}.get(kind, (2000, 256))
    x = rng.normal(size=(n, d)) + rng.normal(size=d) * 2
    if kind == "dead":
        x = np.maximum(x, 0.0)
        x[:, :8] = 0.0
        x[:, 8:12] = 1.5
    elif kind == "duplicated":
        x[:, -32:] = x[:, :32]
    elif kind == "collinear":
        x = rng.integers(-8, 9, size=(n, d)).astype(np.float64)
        x[:, -32:] = x[:, :32] * 2 - x[:, 32:64] + 0.5 * x[:, 64:96]
    elif kind == "constant":
        x[:] = np.round(x[0] * 8) / 8
    return x.astype(dtype)


def scores(x: np.ndarray, ref: dict) -> np.ndarray:
    """Squared Mahalanobis distances of the rows of x, float64: |(x[:, live] - location[live]) . W|^2."""
    live = ref["live"]
    if not live.size:
        return np.zeros(x.shape[0])
    xc = x[:, live].astype(np.float64) - ref["location"][live].astype(np.float64)
    y = xc @ ref["w"]
    return np.sum(y * y, axis=1)


def score_bound(x: np.ndarray, ref: dict, prec_b: float) -> np.ndarray:
    """Per-row bound on |device score - scores(x, ref)|: the precision's error (|xc|^2 prec_b, prec_b being a
    spectral-norm bound), the fp32 whitening (centring, the fp32 factor and a d-term fp32 dot product:
    |dy| <= g |xc| |W_j|, summed by Cauchy-Schwarz into 2 g |xc| sqrt(tr P) sqrt(q) + g^2 |xc|^2 tr P, which does
    not depend on the factor chosen) and the double row norm (4 d u q)."""
    live = ref["live"]
    if not live.size:
        return np.zeros(x.shape[0])
    dl = live.size
    xc = x[:, live].astype(np.float64) - ref["location"][live].astype(np.float64)
    nrm2 = np.sum(xc * xc, axis=1)
    q = scores(x, ref)
    s = ref["eigenvalues"][ref["keep"]]
    tr = float(np.sum(1.0 / s[s > 0]))
    g = gamma(dl + 3, U32)
    return nrm2 * prec_b + 2 * g * np.sqrt(nrm2 * tr * q) + g * g * nrm2 * tr + 4 * dl * U * q
