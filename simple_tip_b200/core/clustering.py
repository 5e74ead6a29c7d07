"""sklearn-compatible k-means and silhouette score on the H100 (the k-means discriminator of MultiModalSA,
surprise.py:102-133).

`KMeans` follows sklearn's `KMeans(init="k-means++", algorithm="lloyd")`: greedy k-means++ seeding,
Lloyd iterations, the best of `n_init` runs by inertia; the draws come from a counter-based RNG keyed by
`random_state`, so results are reproducible bit for bit but are not sklearn's draws.  `silhouette_samples` /
`silhouette_score` follow sklearn.metrics.  X is a NumPy array or a torch CUDA tensor (float32 / float64);
a CUDA tensor never leaves the GPU and the results then stay there too, NumPy input gives NumPy results.
"""
from __future__ import annotations

import numpy as np


def _device_input(X):
    """(device matrix, came-as-tensor flag)"""
    import torch

    from .. import engine as E

    dev = E.require_cuda()
    if isinstance(X, torch.Tensor):
        if not X.is_cuda:
            X = X.to(dev)
        x, is_tensor = X.reshape(X.shape[0], -1), True
    else:
        X = np.asarray(X)
        if X.dtype not in (np.float32, np.float64):
            X = X.astype(np.float64)
        x, is_tensor = E.to_device(X.reshape(X.shape[0], -1), dev), False
    E.tip_dtype(x.dtype)
    return x.contiguous(), is_tensor


def _out(t, is_tensor: bool):
    return t if is_tensor else t.cpu().numpy()


class KMeans:
    """KMeans(n_clusters, n_init=10, max_iter=300, tol=1e-4, random_state=0); attributes as sklearn's:
    cluster_centers_ (X's dtype), labels_ (int32), inertia_, n_iter_."""

    def __init__(self, n_clusters: int = 8, n_init: int = 10, max_iter: int = 300, tol: float = 1e-4,
                 random_state: int = 0):
        from .. import engine as E

        if not (isinstance(n_clusters, (int, np.integer)) and 1 <= n_clusters <= E.KMEANS_MAX_K):
            raise ValueError(f"n_clusters={n_clusters}: the device k-means supports 1 <= n_clusters <= {E.KMEANS_MAX_K}")
        if not 1 <= n_init <= 64:
            raise ValueError(f"n_init={n_init} should be in [1, 64]")
        if max_iter < 1 or tol < 0:
            raise ValueError("max_iter must be >= 1 and tol >= 0")
        self.n_clusters, self.n_init, self.max_iter, self.tol = int(n_clusters), int(n_init), int(max_iter), float(tol)
        self.random_state = int(random_state)

    def fit(self, X, y=None) -> "KMeans":
        from .. import engine as E

        x, is_tensor = _device_input(X)
        if x.shape[0] < self.n_clusters:
            raise ValueError(f"n_samples={x.shape[0]} should be >= n_clusters={self.n_clusters}.")
        cen, labels, inertia, n_iter = E.kmeans_fit(x, self.n_clusters, self.n_init, self.max_iter, self.tol,
                                                    self.random_state)
        self.cluster_centers_, self.labels_ = _out(cen, is_tensor), _out(labels, is_tensor)
        self._centres_dev = cen
        self.inertia_, self.n_iter_ = inertia, n_iter
        return self

    def fit_predict(self, X, y=None):
        return self.fit(X).labels_

    def predict(self, X):
        from .. import engine as E

        x, is_tensor = _device_input(X)
        labels, _ = E.kmeans_predict(x, self._centres_dev)
        return _out(labels, is_tensor)


def _encode_labels(labels, n: int):
    """sklearn's LabelEncoder + check_number_of_labels: labels -> (codes on the device, number of labels)."""
    import torch

    from .. import engine as E

    dev = E.require_cuda()
    lab = labels if isinstance(labels, torch.Tensor) else torch.from_numpy(np.asarray(labels).reshape(-1))
    if lab.shape[0] != n:
        raise ValueError(f"Found input variables with inconsistent numbers of samples: [{n}, {lab.shape[0]}]")
    uniq, codes = torch.unique(lab.to(dev), sorted=True, return_inverse=True)
    n_labels = int(uniq.shape[0])
    if not 1 < n_labels < n:
        raise ValueError(f"Number of labels is {n_labels}. Valid values are 2 to n_samples - 1 (inclusive)")
    return codes, n_labels


def silhouette_samples(X, labels):
    """sklearn.metrics.silhouette_samples (Euclidean): float64 per row."""
    from .. import engine as E

    x, is_tensor = _device_input(X)
    codes, n_labels = _encode_labels(labels, x.shape[0])
    return _out(E.silhouette_samples(x, codes, n_labels), is_tensor)


def silhouette_score(X, labels) -> float:
    """sklearn.metrics.silhouette_score (Euclidean, no sampling): the mean of silhouette_samples, in double."""
    from .. import engine as E

    x, _ = _device_input(X)
    codes, n_labels = _encode_labels(labels, x.shape[0])
    return float(E.silhouette_samples(x, codes, n_labels).mean())
