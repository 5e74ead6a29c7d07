"""sklearn-compatible EmpiricalCovariance fitted on the H100 (the fit of MDSA, surprise.py:374-393).

`EmpiricalCovariance()` follows sklearn 1.9's `EmpiricalCovariance()` (MDSA passes no options):
- `location_ = X.mean(0)` in the input dtype, bit for bit as NumPy computes it (csrc/covariance.cu);
- `covariance_ = np.cov(X.T, bias=1)` in float64, centred on its own float64 mean, as a float64 DMMA scatter
  (csrc/mixture.cu's tip_gmm_scatter with one unit-weight component);
- `precision_ = scipy.linalg.pinvh(covariance_)`: an eigendecomposition (torch.linalg.eigh, float64, on the device)
  with scipy's cutoff |s| > d * eps * max|s|.  Columns whose centred values are all exactly 0 (dead ReLU units,
  constant columns) have an exactly zero row and column; they are left out of the eigendecomposition, so their
  zero eigenvalue is dropped exactly.
`mahalanobis(X)` whitens the live columns with U diag(s^-1/2) in fp32 and sums the squares in double, as MDSA's
scoring always has.  X is a NumPy array or a torch CUDA tensor; a CUDA tensor never leaves the GPU.  Inputs other
than float32 / float64 are widened as MDSA's scoring widens them (host arrays to float64, device tensors to
float32), where sklearn would keep some of them (a documented deviation).
"""
from __future__ import annotations

import warnings

import numpy as np


def _rows(X):
    """(2-D device matrix, came-as-tensor flag); sklearn's errors for empty input are raised before any upload."""
    import torch

    from .surprise import _device_rows

    is_tensor = isinstance(X, torch.Tensor)
    shape = tuple(X.shape) if is_tensor else np.shape(X)
    if len(shape) != 2:
        raise ValueError(f"Expected a 2-dimensional array, got an array of shape {shape}.")
    if shape[0] == 0:
        raise ValueError(f"Found array with 0 sample(s) (shape={shape}) while a minimum of 1 is required by "
                         "EmpiricalCovariance.")
    if shape[1] == 0:
        raise ValueError(f"Found array with 0 feature(s) (shape={shape}) while a minimum of 1 is required by "
                         "EmpiricalCovariance.")
    if is_tensor and not X.is_cuda:
        from .. import engine as E

        X = X.to(E.require_cuda())
    return _device_rows(X if is_tensor else np.asarray(X)), is_tensor


class EmpiricalCovariance:
    """EmpiricalCovariance().  Attributes as sklearn's: location_ (input dtype), covariance_ and precision_ (float64
    NumPy, copied from the device on first access), n_features_in_; plus rank_ (kept eigenvalues)."""

    def fit(self, X, y=None) -> "EmpiricalCovariance":
        from .. import engine as E

        x, _ = _rows(X)
        if x.shape[0] == 1:
            warnings.warn("Only one sample available. You may want to reshape your data array", UserWarning)
        self._dev = E.cov_fit(x)
        self.location_ = self._dev["location"].cpu().numpy()
        self.n_features_in_ = int(x.shape[1])
        self.rank_ = self._dev["rank"]
        self._host = {}
        return self

    def _fitted(self) -> dict:
        if not hasattr(self, "_dev"):
            raise RuntimeError("This EmpiricalCovariance instance is not fitted yet. Call 'fit' first.")
        return self._dev

    def _array(self, key: str) -> np.ndarray:
        fit = self._fitted()
        if key not in self._host:
            self._host[key] = fit[key].cpu().numpy()
        return self._host[key]

    @property
    def covariance_(self) -> np.ndarray:
        return self._array("covariance")

    @property
    def precision_(self) -> np.ndarray:
        return self._array("precision")

    def get_precision(self) -> np.ndarray:
        return self.precision_

    def _scores(self, x):
        """Squared Mahalanobis distances of the rows of the device matrix x, float64 on the device."""
        from .. import engine as E

        fit = self._fitted()
        if x.shape[1] != self.n_features_in_:
            raise ValueError(f"X has {x.shape[1]} features, but EmpiricalCovariance is expecting "
                             f"{self.n_features_in_} features as input.")
        return E.cov_scores(x, fit)

    def mahalanobis(self, X):
        """Squared Mahalanobis distances of the rows of X (float64; a CUDA tensor in gives a CUDA tensor out)."""
        x, is_tensor = _rows(X)
        d = self._scores(x)
        return d if is_tensor else d.cpu().numpy()
