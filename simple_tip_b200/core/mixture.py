"""sklearn-compatible full-covariance Gaussian mixture fitted on the H100 (the density of MLSA, surprise.py:498-520).

`GaussianMixture` follows sklearn's `GaussianMixture(n_components, covariance_type="full", init_params="kmeans",
n_init=1)`: initial responsibilities from the labels of one device k-means run (core/clustering.py's `KMeans` with
n_init=1, seeded by `random_state`, so the start is reproducible bit for bit but is not sklearn's), then EM until
the lower bound changes by less than `tol`.  Every N-sized pass runs in float64 on the fp64 tensor cores
(csrc/mixture.cu); the d x d factorisations run batched on the device (torch.linalg, float64).  X is a NumPy array
or a torch CUDA tensor (float32 / float64); a CUDA tensor never leaves the GPU.  The fitted attributes carry
sklearn's names and are float64 NumPy arrays, whatever the input dtype.
"""
from __future__ import annotations

import warnings

import numpy as np

from .clustering import _device_input, _out

MAX_COMPONENTS = 64     # the device k-means limit


def _n_samples(X) -> int:
    shape = tuple(X.shape) if hasattr(X, "shape") else np.shape(X)
    return int(shape[0]) if len(shape) else 0


class GaussianMixture:
    """GaussianMixture(n_components=1, tol=1e-3, reg_covar=1e-6, max_iter=100, random_state=0).  Attributes as
    sklearn's: weights_, means_, covariances_, precisions_cholesky_ (float64 NumPy), converged_, n_iter_,
    lower_bound_, lower_bounds_, covariance_type = "full"."""

    covariance_type = "full"

    def __init__(self, n_components: int = 1, tol: float = 1e-3, reg_covar: float = 1e-6, max_iter: int = 100,
                 random_state: int = 0):
        if not (isinstance(n_components, (int, np.integer)) and 1 <= n_components <= MAX_COMPONENTS):
            raise ValueError(f"n_components={n_components}: the device mixture supports "
                             f"1 <= n_components <= {MAX_COMPONENTS}")
        if not (isinstance(max_iter, (int, np.integer)) and max_iter >= 1):
            raise ValueError(f"max_iter={max_iter} must be an integer >= 1")
        if not tol >= 0:
            raise ValueError(f"tol={tol} must be >= 0")
        if not reg_covar >= 0:
            raise ValueError(f"reg_covar={reg_covar} must be >= 0")
        self.n_components, self.max_iter = int(n_components), int(max_iter)
        self.tol, self.reg_covar, self.random_state = float(tol), float(reg_covar), int(random_state)

    def fit(self, X, y=None) -> "GaussianMixture":
        from .. import engine as E

        n = _n_samples(X)
        if n < 2:
            raise ValueError(f"Found array with {n} sample(s) while a minimum of 2 is required by GaussianMixture.")
        if n < self.n_components:
            raise ValueError("Expected n_samples >= n_components "
                             f"but got n_components = {self.n_components}, n_samples = {n}")
        x, _ = _device_input(X)
        fit = E.gmm_fit(x, self.n_components, self.max_iter, self.tol, self.reg_covar, self.random_state)
        self._set_state(fit["weights"], fit["means"], fit["prec_chol"], fit["log_det"])
        self.covariances_ = fit["covariances"].cpu().numpy()
        self.labels_init_ = fit["labels_init"]
        self.converged_, self.n_iter_ = bool(fit["converged"]), int(fit["n_iter"])
        self.lower_bound_, self.lower_bounds_ = float(fit["lower_bound"]), list(fit["lower_bounds"])
        if not self.converged_:
            from sklearn.exceptions import ConvergenceWarning

            warnings.warn("Best performing initialization did not converge. Try different init parameters, or "
                          "increase max_iter, tol, or check for degenerate data.", ConvergenceWarning)
        return self

    def _set_state(self, weights, means, prec_chol, log_det):
        self._dev = (weights, means, prec_chol, log_det)
        self.weights_ = weights.cpu().numpy()
        self.means_ = means.cpu().numpy()
        self.precisions_cholesky_ = prec_chol.cpu().numpy()
        self.n_features_in_ = int(self.means_.shape[1])

    def _estimate(self, X, **want):
        import torch

        from .. import engine as E

        if not hasattr(self, "_dev"):
            raise RuntimeError("This GaussianMixture instance is not fitted yet. Call 'fit' first.")
        x, is_tensor = _device_input(X)
        if x.shape[1] != self.n_features_in_:
            raise ValueError(f"X has {x.shape[1]} features, but GaussianMixture is expecting {self.n_features_in_} "
                             "features as input.")
        weights, means, prec_chol, log_det = self._dev
        q = E.gmm_quad(x, means, prec_chol)
        return E.gmm_resp(q, x.shape[1], torch.log(weights), log_det, **want), is_tensor

    def score_samples(self, X):
        """Per-row log-likelihood (float64), sklearn's score_samples."""
        (_, lse, _, _), is_tensor = self._estimate(X, want_resp=False, want_lse=True)
        return _out(lse, is_tensor)

    def score(self, X, y=None) -> float:
        return float(self.score_samples(X).mean())

    def predict(self, X):
        """The most probable component of every row (int64), sklearn's predict."""
        (_, _, labels, _), is_tensor = self._estimate(X, want_resp=False, want_labels=True)
        return _out(labels, is_tensor)

    def predict_proba(self, X):
        (resp, _, _, _), is_tensor = self._estimate(X, want_resp=True)
        return _out(resp.t().contiguous(), is_tensor)

    def fit_predict(self, X, y=None):
        return self.fit(X).predict(X)
