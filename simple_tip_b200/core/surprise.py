"""Surprise adequacies behind the reference's `src.core.surprise` API, scored on an H100.

Drop-in for `/root/reference/src/core/surprise.py`: same class names, constructor = fit,
`__call__` = score, same argument meaning, same assertion / error messages
(tests/test_surprise.py of the reference runs against this module through the `src/core`
overlay).  The pair arithmetic of DSA and LSA runs in libb200tip.so (wgmma filter + exact
re-rank, fused KDE log-sum-exp); everything that decides WHICH rows are compared (flattening,
label validation, seeded sub-sampling, class grouping, column selection, the float64 KDE fit)
stays host NumPy with the reference's expressions.  `fit` / `score` are additive aliases.
"""
from __future__ import annotations

import abc
import os
import warnings
from typing import Callable, Dict, Iterable, List, Optional, Tuple, Union

import numpy as np

from .stable_kde import StableGaussianKDE

Activations = Union[List[np.ndarray], np.ndarray]
Predictions = Union[List[Union[int, float]], np.ndarray]
Discriminator = Callable[[Activations, Predictions], np.ndarray]


# ------------------------------------------------------------------------------------------
# input normalisation (reference: surprise.py:55-87, 136-183) — host side, bit-for-bit
# ------------------------------------------------------------------------------------------
def _subsample_arrays(subsampling: Union[int, float], arrays: Tuple[np.ndarray, ...], seed: int
                      ) -> Tuple[np.ndarray, ...]:
    """Same rows for every array; `RandomState(seed).choice(arange(n), k, replace=False)`
    exactly as surprise.py:84-86 so that the SAME training rows enter the kernel."""
    n = arrays[0].shape[0]
    assert all(a.shape[0] == n for a in arrays), "All arrays must have the same number of samples"
    if subsampling == 1.0:
        return arrays
    if isinstance(subsampling, int) and subsampling > 0:
        k = min(subsampling, n)
    elif 0 < subsampling < 1:
        k = int(subsampling * n)
    else:
        raise ValueError(
            "subsampling must be a float between 0 and 1 (share of training data),"
            "or a positive int declaring the number of samples")
    picked = np.random.RandomState(seed).choice(np.arange(n), k, replace=False)
    return tuple(_take_rows(a, picked) for a in arrays)


def _take_rows(a, rows: np.ndarray):
    """a[rows] for NumPy arrays and for device-resident traces (torch tensors)."""
    if isinstance(a, np.ndarray):
        return a[rows]
    import torch

    return a.index_select(0, torch.from_numpy(np.asarray(rows, dtype=np.int64)).to(a.device))


def _subsample_array(subsampling, array: np.ndarray, seed: int) -> np.ndarray:
    return _subsample_arrays(subsampling, (array,), seed=seed)[0]


def _class_predictions(predictions: Predictions, num_classes: int = None) -> np.ndarray:
    """1-D integer class ids; messages pinned by the reference's tests/test_surprise.py:33-45."""
    if isinstance(predictions, list):
        predictions = np.array(predictions)
    assert predictions.ndim == 1, (
        "Class predictions must be one-dimensional. "
        "If your predictions are one_hot encoded, use eg `np.argmax(softmax_outputs, axis=1)`")
    if predictions.dtype != np.dtype(int):
        np.testing.assert_almost_equal(predictions, predictions.astype(int), decimal=5,
                                       err_msg="Predictions must be integers")
        predictions = predictions.astype(int)
    assert np.all(predictions >= 0), "Class predictions must be >= 0"
    assert num_classes is None or np.all(predictions < num_classes), "Class predictions must be < num_classes"
    return predictions


def _flatten_layers(layers: Activations) -> np.ndarray:
    if isinstance(layers, np.ndarray):
        return layers if layers.ndim == 2 else layers.reshape((layers.shape[0], -1))
    return np.concatenate([np.reshape(l, (l.shape[0], -1)) for l in layers], axis=1)


def _flatten_predictions(predictions: Predictions) -> Optional[np.ndarray]:
    if predictions is None:
        return None
    return predictions if isinstance(predictions, np.ndarray) else np.array(predictions)


def _by_class_discriminator(activations: Activations, predictions: Predictions) -> np.ndarray:
    return _class_predictions(predictions)


def _kmeans_backend(backend: Optional[str]) -> str:
    """backend=None: the B200TIP_KMEANS environment variable, default "sklearn"."""
    backend = backend if backend is not None else os.environ.get("B200TIP_KMEANS", "sklearn")
    if backend not in ("sklearn", "device"):
        raise ValueError(f"backend must be 'sklearn' or 'device', got {backend!r}")
    return backend


def _gmm_backend(backend: Optional[str]) -> str:
    """backend=None: the B200TIP_GMM environment variable, default "sklearn"."""
    backend = backend if backend is not None else os.environ.get("B200TIP_GMM", "sklearn")
    if backend not in ("sklearn", "device"):
        raise ValueError(f"backend must be 'sklearn' or 'device', got {backend!r}")
    return backend


def _cov_backend(backend: Optional[str]) -> str:
    """backend=None: the B200TIP_COV environment variable, default "sklearn"."""
    backend = backend if backend is not None else os.environ.get("B200TIP_COV", "sklearn")
    if backend not in ("sklearn", "device"):
        raise ValueError(f"backend must be 'sklearn' or 'device', got {backend!r}")
    return backend


def _kde_backend(backend: Optional[str]) -> str:
    """backend=None: the B200TIP_KDE environment variable, default "host"."""
    backend = backend if backend is not None else os.environ.get("B200TIP_KDE", "host")
    if backend not in ("host", "device"):
        raise ValueError(f"backend must be 'host' or 'device', got {backend!r}")
    return backend


def _trace_matrix(activations):
    """[N, D] traces: the device matrix for torch CUDA traces, else the reference's host flattening."""
    from .. import engine as E

    x = E.device_matrix(activations)
    return x if x is not None else _flatten_layers(activations)


def _host_matrix(activations) -> np.ndarray:
    """[N, D] host traces: torch CUDA traces downloaded once, else the reference's host flattening."""
    from .. import engine as E

    x = E.device_matrix(activations)
    return x.cpu().numpy() if x is not None else _flatten_layers(activations)


class _KmeansDiscriminator:
    """k-means modal assignment with silhouette model selection (surprise.py:102-133).
    backend="sklearn" (default): sklearn on the host, as the reference; torch CUDA traces are downloaded once per
    call.  backend="device": k-means and the silhouette score on the GPU (core/clustering.py), seeded with
    `random_state` (the reference's sklearn call is unseeded); CUDA traces stay on the device."""

    def __init__(self, training_data: Activations, potential_k: Iterable[int], subsampling=1.0,
                 subsampling_seed: int = 0, n_init: int = 10, max_iter: int = 300, backend: Optional[str] = None,
                 random_state: int = 0):
        self.backend = _kmeans_backend(backend)
        if self.backend == "device":
            from .. import engine as E
            from .clustering import KMeans, silhouette_score

            E.require_cuda()
            data = _subsample_array(subsampling, _trace_matrix(training_data), seed=subsampling_seed)
        else:
            from sklearn.cluster import KMeans
            from sklearn.metrics import silhouette_score

            data = _subsample_array(subsampling, _host_matrix(training_data), seed=subsampling_seed)
        self.best_score, self.best_k, self.best_clusterer = -np.inf, None, None
        for k in potential_k:
            if self.backend == "device":
                km = KMeans(n_clusters=k, n_init=n_init, max_iter=max_iter, random_state=random_state)
            else:
                km = KMeans(n_clusters=k, n_init=n_init, max_iter=max_iter)
            score = silhouette_score(data, km.fit_predict(data))
            if score > self.best_score:
                self.best_score, self.best_k, self.best_clusterer = score, k, km

    def __call__(self, activations: Activations, predictions: Predictions) -> np.ndarray:
        if self.backend == "device":
            from .. import engine as E

            return E.host_array(self.best_clusterer.predict(_trace_matrix(activations)))
        return self.best_clusterer.predict(_host_matrix(activations))


class SurpriseCoverageMapper:
    """SA value -> one-hot bucket profile over [0, upper_bound] (surprise.py:186-209)."""

    def __init__(self, sections: int, upper_bound: float, overflow_bucket: bool = False):
        self.sections, self.upper_bound = sections, upper_bound
        edges = np.linspace(start=0, stop=upper_bound, num=sections if overflow_bucket else sections + 1,
                            dtype=np.float64)
        self.thresholds = np.concatenate((edges, [np.inf])) if overflow_bucket else edges

    def get_coverage_profile(self, surprise_values: np.ndarray) -> np.ndarray:
        lo, hi = self.thresholds[:-1], self.thresholds[1:]
        v = np.asarray(surprise_values)[..., None]
        return np.logical_and(lo <= v, v < hi)


class SA(abc.ABC):
    def __init__(self):
        super().__init__()

    @abc.abstractmethod
    def __call__(self, activations: Activations, predictions: Predictions, num_threads: int = 1) -> np.ndarray:
        ...

    def score(self, activations, predictions=None, **kw) -> np.ndarray:
        return self(activations, predictions, **kw)

    def score_begin(self, activations, predictions=None):
        """Start scoring and return an object whose `finish()` yields the scores.  Default: score synchronously.
        Scorers that can keep their kernels and the result copy in flight override this (LSA)."""
        return _Finished(self(activations, predictions))

    @classmethod
    def fit(cls, *args, **kw):
        return cls(*args, **kw)


class _Finished:
    def __init__(self, value):
        self.value = value

    def finish(self):
        return self.value


class MultiModalSA(SA):
    """Routes every sample to the SA of its modal (surprise.py:226-371)."""

    def __init__(self, discriminator: Discriminator, modal_sa: Dict[int, SA]):
        super().__init__()
        self.discriminator, self.modal_sa = discriminator, modal_sa

    @staticmethod
    def build_by_class(activations, predictions, sa_constructor) -> "MultiModalSA":
        return MultiModalSA.build(activations, predictions, _by_class_discriminator, sa_constructor)

    @staticmethod
    def build_with_kmeans(activations, predictions, sa_constructor, potential_k: Iterable[int], n_init: int = 10,
                          max_iter: int = 300, subsampling=1.0, subsampling_seed: int = 0,
                          backend: Optional[str] = None, random_state: int = 0) -> "MultiModalSA":
        """backend / random_state: see _KmeansDiscriminator (B200TIP_KMEANS=device selects the GPU backend)."""
        disc = _KmeansDiscriminator(activations, potential_k, n_init=n_init, max_iter=max_iter,
                                    subsampling=subsampling, subsampling_seed=subsampling_seed, backend=backend,
                                    random_state=random_state)
        if disc.backend == "device":
            activations = _host_matrix(activations)      # the modal SAs are fitted on host rows, as the reference does
        return MultiModalSA.build(activations, predictions, disc, sa_constructor)

    @staticmethod
    def build(activations, predictions, discriminator: Discriminator, sa_constructor) -> "MultiModalSA":
        """CUDA traces (one tensor or a list of hook layers) are split by modal on the device, and the constructors
        receive CUDA tensors; NumPy traces are split on the host, as the reference does."""
        from .. import engine as E

        x = E.device_matrix(activations)
        if x is not None:
            preds = _flatten_predictions(E.host_array(predictions))
            modal = E.host_array(discriminator(x, preds))
            fitted: Dict[int, SA] = {}
            for mid in np.unique(modal):
                rows = np.flatnonzero(modal == mid)
                fitted[mid] = sa_constructor(_take_rows(x, rows), None if preds is None else preds[rows])
            return MultiModalSA(discriminator=discriminator, modal_sa=fitted)
        acts = _flatten_layers(activations)
        preds = _flatten_predictions(predictions)
        modal = discriminator(acts, preds)
        fitted: Dict[int, SA] = {}
        for mid in np.unique(modal):
            rows = modal == mid
            fitted[mid] = sa_constructor(acts[rows], None if preds is None else preds[rows])
        return MultiModalSA(discriminator=discriminator, modal_sa=fitted)

    def _get_sa_for_modal_id(self, modal_id: int) -> SA:
        try:
            return self.modal_sa[modal_id]
        except KeyError:
            raise ValueError(f"No modal found for modal id {modal_id}. Check your discriminator")

    def __call__(self, activations, predictions, num_threads: int = 1) -> np.ndarray:
        """CUDA traces (one tensor or a list of hook layers) are split by modal on the device, whatever the
        discriminator; NumPy traces are flattened on the host, as the reference does."""
        from .. import engine as E

        predictions = E.host_array(predictions)
        modal = self.discriminator(activations, predictions)
        acts = _trace_matrix(activations)
        preds = _flatten_predictions(predictions)
        assert len(modal) == acts.shape[0], (
            f"The discriminator returned an invalid number ({len(modal)}) of modal indexes."
            f"Expected: {acts.shape[0]} indexes.")
        if len(modal) == 0:
            return np.ndarray(shape=(0,))
        present = np.unique(modal)
        sas = [self._get_sa_for_modal_id(mid) for mid in present]
        # One CUDA stream serves all modals (the reference's thread pool, surprise.py:345, only overlapped CPU
        # work).  The traces are uploaded ONCE and split by modal on the device; every modal's kernels and its
        # result copy are launched before the first result is waited for (`score_begin` / `finish`).
        per_modal = None
        ours = all(isinstance(sa, (LSA, MDSA, MLSA, DSA)) for sa in sas)    # user-defined SAs keep getting NumPy arrays
        float_rows = not isinstance(acts, np.ndarray) or acts.dtype in (np.float32, np.float64)   # device traces: checked later
        if ours and float_rows and len(present) > 1:
            try:
                import torch

                from .. import engine as E

                dev = E.require_cuda()
                order = np.argsort(modal, kind="stable")
                counts = [int(np.count_nonzero(modal == mid)) for mid in present]
                x_sorted = E.to_device(acts, dev).index_select(0, torch.from_numpy(order).to(dev))
                pending, lo = [], 0
                for sa, mid, cnt in zip(sas, present, counts):
                    rows = order[lo:lo + cnt]
                    pending.append(sa.score_begin(x_sorted[lo:lo + cnt], None if preds is None else preds[rows]))
                    lo += cnt
                per_modal = [p.finish() for p in pending]
            except RuntimeError as e:
                if "CUDA device" not in str(e):
                    raise
                per_modal = None      # no GPU: let the per-modal calls raise their own (loud) error below
        if per_modal is None:
            per_modal = []
            for sa, mid in zip(sas, present):
                rows = modal == mid
                sel = acts[rows] if isinstance(acts, np.ndarray) else _take_rows(acts, np.flatnonzero(rows))
                per_modal.append(sa(sel, None if preds is None else preds[rows], num_threads=num_threads))
        res = np.full(fill_value=-np.inf, shape=modal.shape, dtype=per_modal[0].dtype)
        for mid, vals in zip(present, per_modal):
            res[modal == mid] = vals
        return res


def _psd_factor(precision: np.ndarray) -> np.ndarray:
    """W with W . W^T = precision for a symmetric positive SEMI-definite matrix (float64, host): eigenvectors
    scaled by the square roots of the (clipped) eigenvalues, so |(x - mu) . W|^2 = (x - mu)^T P (x - mu) also when
    sklearn's pinvh produced a singular precision."""
    vals, vecs = np.linalg.eigh((precision + precision.T) / 2.0)
    return vecs * np.sqrt(np.clip(vals, 0.0, None))[None, :]


def _device_rows(activations):
    """[N, D] device matrix (float32 / float64) from NumPy arrays, lists of layers or torch CUDA tensors."""
    import torch

    from .. import engine as E

    dev = E.require_cuda()
    x = E.device_matrix(activations)
    if x is None:
        a = _flatten_layers(activations)
        if a.dtype not in (np.float32, np.float64):
            a = a.astype(np.float64)
        x = E.to_device(a, dev)
    elif x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float32)
    return x.contiguous()


class MDSA(SA):
    """Mahalanobis-distance surprise adequacy (surprise.py:374-393): squared Mahalanobis distance to the mean of
    the training traces.  Fit = sklearn's `EmpiricalCovariance` on the host exactly as in the reference (one
    D x D covariance, its pseudo-inverse); score = whitening by a factor of the precision + squared row norm on
    the GPU (tip_whiten + tip_row_sqnorm), float64 out like `EmpiricalCovariance.mahalanobis`.
    backend="sklearn" (default, or B200TIP_COV unset): the fit is sklearn's on the host.  backend="device": the fit
    runs on the GPU (core/covariance.py: sklearn's location_ bit for bit, the covariance and its pseudo-inverse in
    float64); CUDA traces then stay on the device, and the whitening factor comes from the fit's own
    eigendecomposition over the live columns."""

    def __init__(self, activations: Activations, *, backend: Optional[str] = None):
        super().__init__()
        from .. import engine as E

        self.backend = _cov_backend(backend)
        if self.backend == "device":
            from .covariance import EmpiricalCovariance

            E.require_cuda()
            acts = _trace_matrix(activations)
        else:
            from sklearn.covariance import EmpiricalCovariance

            acts = _host_matrix(activations)
        self.covariance_matrix = EmpiricalCovariance()
        self.covariance_matrix.fit(acts)
        self._width = int(acts.shape[1])
        self._centres = None

    def _upload(self):
        import torch

        from .. import engine as E

        dev = E.require_cuda()
        w = _psd_factor(np.asarray(self.covariance_matrix.get_precision(), dtype=np.float64))
        mu = np.asarray(self.covariance_matrix.location_, dtype=np.float64)
        self._centres = [(torch.from_numpy(mu).to(dev), torch.from_numpy(np.ascontiguousarray(w.astype(np.float32))).to(dev))]

    def __call__(self, activations, predictions=None, num_threads=None) -> np.ndarray:
        from .. import engine as E

        x = _device_rows(activations)
        if x.ndim != 2 or int(x.shape[1]) != self._width:
            raise ValueError(f"X has {tuple(x.shape)[1:]} features, but MDSA was fitted with {self._width} features")
        if self.backend == "device":
            return self.covariance_matrix._scores(x).cpu().numpy()
        if self._centres is None:
            self._upload()
        return E.quadratic_forms(x, self._centres)[0].cpu().numpy()


class MLSA(SA):
    """Multimodal likelihood surprise adequacy (surprise.py:498-520): negative log-likelihood under a Gaussian
    mixture.  Fit = sklearn's `GaussianMixture` on the host as in the reference; score: per component
    y = (x - mu_k) . precisions_cholesky_k on the GPU (sklearn `_estimate_log_gaussian_prob`), squared row norms,
    then `-logsumexp_k(log w_k - (D log 2pi + |y|^2) / 2 + log det chol_k)` in float64 on the host — the tail of
    `GaussianMixture.score_samples`.
    backend="sklearn" (default, or B200TIP_GMM unset): the fit is sklearn's on the host.  backend="device": the fit
    runs on the GPU in float64 (core/mixture.py), its k-means start seeded with `random_state` (the reference's
    sklearn call is unseeded); CUDA traces then stay on the device.  Scoring is the same for both."""

    def __init__(self, activations: Activations, num_components: int = 2, *, backend: Optional[str] = None,
                 random_state: int = 0):
        super().__init__()
        from .. import engine as E

        self.backend = _gmm_backend(backend)
        if self.backend == "device":
            from .mixture import GaussianMixture

            E.require_cuda()
            acts = _trace_matrix(activations)
            self.gmm = GaussianMixture(n_components=num_components, random_state=random_state)
        else:
            from sklearn.mixture import GaussianMixture

            acts = _host_matrix(activations)
            self.gmm = GaussianMixture(n_components=num_components)
        self.gmm.fit(acts)
        self._width = int(acts.shape[1])
        self._centres = None

    def _upload(self):
        import torch

        from .. import engine as E

        dev = E.require_cuda()
        if self.gmm.covariance_type != "full":
            raise NotImplementedError("only sklearn's default covariance_type='full' (what the reference uses)")
        chol = np.asarray(self.gmm.precisions_cholesky_, dtype=np.float64)
        self._centres = [(torch.from_numpy(np.ascontiguousarray(self.gmm.means_[k], dtype=np.float64)).to(dev),
                          torch.from_numpy(np.ascontiguousarray(chol[k].astype(np.float32))).to(dev))
                         for k in range(chol.shape[0])]
        # log det of the precision Cholesky factors (sklearn _compute_log_det_cholesky, 'full')
        self._log_det = np.array([np.sum(np.log(np.diag(chol[k]))) for k in range(chol.shape[0])])
        self._log_w = np.log(np.asarray(self.gmm.weights_, dtype=np.float64))

    def __call__(self, activations, predictions=None, num_threads=0) -> np.ndarray:
        from scipy.special import logsumexp

        from .. import engine as E

        x = _device_rows(activations)
        if x.ndim != 2 or int(x.shape[1]) != self._width:
            raise ValueError(f"X has {tuple(x.shape)[1:]} features, but MLSA was fitted with {self._width} features")
        if self._centres is None:
            self._upload()
        q = E.quadratic_forms(x, self._centres).cpu().numpy()            # [K, m]
        log_prob = -0.5 * (self._width * np.log(2 * np.pi) + q) + self._log_det[:, None]
        return -logsumexp(log_prob + self._log_w[:, None], axis=0)


# ------------------------------------------------------------------------------------------
# LSA
# ------------------------------------------------------------------------------------------
class LSA(SA):
    """Likelihood-based surprise adequacy (surprise.py:396-495).

    fit: highest-variance column selection (:417-434) and the float64 KDE fit of
    `StableGaussianKDE`; score: whitening + fused Gaussian-KDE log-sum-exp on the
    GPU, then `-np.log(density)` (:494-495; +inf where the float64 density underflows to 0).
    backend="host" (default, or B200TIP_KDE unset): the fit is the reference's host NumPy.  backend="device": np.var
    bit for bit (tip_col_var), the covariance, its factorisations and the training-row whitening in float64 on the
    GPU (StableGaussianKDE.from_device); the column selection stays the reference's host expression, run on the
    downloaded variances.  Traces may be torch CUDA tensors under either backend (the host backend downloads them);
    bf16 / fp16 CUDA traces are widened to float32."""

    def __init__(self, activations: Activations, var_threshold: Optional[float] = None,
                 max_features: Optional[Union[int, float]] = 300, *, comm=None, backend: Optional[str] = None):
        super().__init__()
        import torch

        from .. import engine as E

        self._comm = comm         # additive: N_train-sharded KDE evaluation (engine.TrainShardComm)
        self.backend = _kde_backend(backend)
        if self.backend == "device" and comm is not None and comm.world > 1:
            raise NotImplementedError("the device KDE fit is not sharded over N_train; use backend='host' with comm")
        dev = E.device_matrix(activations)
        if dev is not None and dev.dtype not in (torch.float32, torch.float64):
            dev = dev.float()
        if self.backend == "device":
            E.require_cuda()
            activations = _device_rows(activations if dev is None else dev)
            var_dev, self._mean, _ = E.col_var(activations)
            var = var_dev.cpu().numpy()
            variances = lambda: var       # noqa: E731  (identical bits to np.var(activations, axis=0))
        else:
            activations = dev.cpu().numpy() if dev is not None else _flatten_layers(activations)
            variances = lambda: np.var(activations, axis=0)       # noqa: E731
        self._source_width = int(activations.shape[1])
        assert var_threshold is None or max_features is None, (
            "Both var_threshold and max_features cannot be specified at the same time."
            "We recommend using the max_features arg to dynamically keep the features"
            "with the highest variance.")
        self.removed_neurons: List[int]
        if var_threshold is not None and var_threshold > 0:
            self.removed_neurons = np.where(variances() < var_threshold)[0]
        if max_features is not None:
            width = activations.shape[1]
            keep = min(max_features * width, width) if max_features < 1 else min(max_features, width)
            self.removed_neurons = [int(c) for c in np.argsort(variances())[:-keep]]
        self.kde = self._create_gaussian_kde(activations)

    def _create_gaussian_kde(self, activations):
        if self.backend == "device":
            kept = np.delete(np.arange(activations.shape[1]), self.removed_neurons)
            if kept.size == 0:
                warnings.warn("All activation traces were removed (variance filter); this LSA instance "
                              "will always report density 0", UserWarning)
                self.kde = None
                return None
            try:
                return StableGaussianKDE.from_device(activations, kept if len(self.removed_neurons) > 0 else None,
                                                     self._mean)
            except (np.linalg.LinAlgError, ValueError) as e:
                # the device fit raises neither of the two messages the reference retries on (see below)
                warnings.warn("Problem regarding KDE fitting", UserWarning)
                raise e
        cleaned = self._remove_unused_columns(activations)
        if cleaned.shape[1] == 0:
            warnings.warn("All activation traces were removed (variance filter); this LSA instance "
                          "will always report density 0", UserWarning)
            self.kde = None
            return None
        try:
            kept = np.delete(np.arange(activations.shape[1]), self.removed_neurons) \
                if len(self.removed_neurons) > 0 else None
            return StableGaussianKDE(cleaned.transpose(), source_columns=kept, comm=self._comm)
        except (np.linalg.LinAlgError, ValueError) as e:
            # surprise.py:456-476: only two message patterns trigger drop-a-neuron-and-retry;
            # NumPy's "Matrix is not positive definite" matches neither, so this re-raises.
            import re

            text = str(e)
            if ("-th leading minor of the array is not positive definite" in text
                    or "numerical imprecision in covariance matrix" in text):
                bad_row = int(re.findall("\\d*", text)[0]) - 1
                bad = np.delete(np.arange(activations.shape[1]), self.removed_neurons)[bad_row]
                warnings.warn(f"Dropping AT {bad}, as leading to numerical error.", UserWarning, 1)
                self.removed_neurons.append(bad)
                return self._create_gaussian_kde(activations)
            warnings.warn("Problem regarding KDE fitting", UserWarning)
            raise e

    def _remove_unused_columns(self, tr_activations):
        if self.removed_neurons is not None and len(self.removed_neurons) > 0:
            return np.delete(tr_activations, self.removed_neurons, axis=1)
        return tr_activations

    def __call__(self, activations, predictions=None, num_threads: int = 0) -> np.ndarray:
        return self.score_begin(activations, predictions).finish()

    def score_begin(self, activations, predictions=None):
        from .. import engine as E

        dev = E.device_matrix(activations)            # traces already in HBM stay there
        activations = dev if dev is not None else _flatten_layers(activations)
        if activations.ndim != 2 or int(activations.shape[1]) != self._source_width:
            # the reference fails here too (np.delete IndexError / scipy's dimension ValueError); the
            # kernels index with the fitted columns, so a narrower matrix must never reach them
            raise ValueError(f"activation traces have {tuple(activations.shape)[1:]} features per sample, "
                             f"this LSA was fitted on {self._source_width}")
        if self.kde is None:
            return _Finished(np.zeros(shape=(activations.shape[0],)))
        # column removal happens on the GPU (the kde knows which source columns it was fitted on)
        return _PendingLsa(self.kde.evaluate_rows_begin(activations))


class _PendingLsa:
    def __init__(self, pending_density):
        self.pending = pending_density

    def finish(self) -> np.ndarray:
        density = self.pending.finish()
        with np.errstate(divide="ignore"):
            return -np.log(density)                  # surprise.py:494-495


# ------------------------------------------------------------------------------------------
# DSA
# ------------------------------------------------------------------------------------------
class DSA(SA):
    """Distance-based surprise adequacy (surprise.py:523-691).

    dsa = dist_a / dist_b with dist_a the distance from the test trace to the nearest training
    trace of its predicted class and dist_b the distance from THAT TRAINING TRACE to the nearest
    training trace of any other class (surprise.py:615-631).  Distances and the winner are
    bit-identical to the reference's NumPy (`np.linalg.norm(axis=2)`, `np.argmin`).

    dtypes: float32 and float64 traces are scored in their own dtype; float64 test traces against float32 training
    traces are scored in float64 like NumPy's promotion does (a float64 twin of the engine is built on first use);
    float16 / bfloat16 traces are widened exactly and scored in float32 (the reference would keep float16
    arithmetic — a documented deviation, INTEGRATION.md)."""

    def __init__(self, activations: Activations, predictions: Predictions, badge_size: int = 10,
                 subsampling: Union[int, float] = 1.0, subsampling_seed: int = 0, *, comm=None):
        super().__init__()
        from .. import engine as E

        # traces may already live in HBM (torch CUDA tensors, e.g. from a forward hook): they stay there
        dev_train = E.device_matrix(activations)
        self.train_activations = dev_train if dev_train is not None else _flatten_layers(activations)
        self.train_predictions: np.ndarray = _class_predictions(E.host_array(predictions))
        self.train_activations, self.train_predictions = _subsample_arrays(
            subsampling, (self.train_activations, self.train_predictions), subsampling_seed)
        self.num_classes = np.max(self.train_predictions) + 1
        self.class_matrix = self._class_matrix()
        self.badge_size = badge_size          # kept for API compatibility; tiles replace badges
        self.use_filter = os.environ.get("B200TIP_DSA_EXHAUSTIVE", "0") != "1"
        self.use_graphs = E.GRAPHS            # CUDA-graph replay of the search
        self.capture_on_first_call = False
        self._seen_shapes = E.BoundedCache(65)
        self._comm = comm
        self._engine = None
        self._engine_wide = None      # float64 twin for float64 test traces against float32 training traces
        self._last_dtype = None
        self._build_engine()

    def _class_matrix(self) -> List[np.ndarray]:
        return [np.argwhere(self.train_predictions == c).flatten() for c in range(self.num_classes)]

    def fit_other_class_table(self) -> "DSA":
        """Extension (not in the reference): tabulate, once per training set, every train row's distance to its
        nearest row of another class.  dist_b of surprise.py:622-631 depends on the test input only through which
        train row won stage 1, so later calls run stage 1 alone and look dist_b up — same bits, N_train x N_train
        pairs moved from every call into the fit.  Single-GPU engines only; drop_other_class_table() reverts."""
        if self._comm is not None and self._comm.world > 1:
            raise NotImplementedError("fit_other_class_table: not available for an N_train-sharded DSA")
        self._engine.build_other_class_table()
        self._seen_shapes.clear()
        return self

    def drop_other_class_table(self) -> "DSA":
        self._engine.table_b = None
        self._seen_shapes.clear()
        return self

    def _build_engine(self):
        from .. import engine as E

        train = self.train_activations
        if isinstance(train, np.ndarray):
            if train.dtype not in (np.float32, np.float64):
                train = train.astype(np.result_type(train.dtype, np.float32))
            self._compute_dtype = train.dtype
        else:       # device tensor: float64 stays, everything else is scored in float32
            self._compute_dtype = np.dtype(np.float64) if str(train.dtype) == "torch.float64" else np.dtype(np.float32)
        labels = self.train_predictions
        if self._comm is not None and self._comm.world > 1:
            # N_train sharded: every class is dealt round-robin over the ranks; the raw training set stays
            # replicated in HBM (original row order) so that global stage-1 winners are gathered by index
            import torch

            dev = E.require_cuda()
            full = E.to_device(train, dev)
            if full.dtype not in (torch.float32, torch.float64):
                full = full.to(torch.float32)
            keep = E.shard_rows(labels, int(self.num_classes), self._comm.rank, self._comm.world)
            shard = full.index_select(0, torch.from_numpy(keep).to(dev))
            self._engine = E.NnEngine.from_host(shard, labels[keep], int(self.num_classes), keep, seeds=False)
            self._engine.t_full = full.contiguous()
        else:
            self._engine = E.NnEngine.from_host(train, labels, int(self.num_classes), np.arange(train.shape[0]))

    def __call__(self, activations: Activations, predictions: Predictions, num_threads: int = None) -> np.ndarray:
        import torch

        from .. import engine as E

        x_all, order, q_off, labels, promoted = self._prepare(activations, predictions)
        n_total, eng = labels.shape[0], self._engine
        if order.size == 0:       # no row to score
            self._last_raw = np.full((4, n_total), np.nan)
            self._last_raw[2] = -1.0
            return self._last_raw[3].copy()
        comm = self._comm if (self._comm is not None and self._comm.world > 1) else None
        # A batch shape (size, class histogram) seen for the first time is launched eagerly — the reference's
        # pipeline scores most datasets exactly once (handler_surprise.py:84-99) and a capture costs ~3 eager
        # calls; its CUDA-graph plan is captured on the second sighting and replayed from then on.
        shape_key = (int(order.size), n_total, q_off.tobytes(), str(x_all.dtype))
        if not promoted and self.use_graphs and (self.capture_on_first_call or self._seen_shapes.touch(shape_key)):
            # steady state: upload the permutation, replay, one D2H copy into pinned memory
            plan = E.dsa_plan(eng, int(order.size), q_off, x_all.dtype, self.use_filter, comm, n_total=n_total)
            if plan.x_in.data_ptr() != x_all.data_ptr():
                # the engine recycled its landing buffer since this plan was captured (many batch sizes)
                plan.x_in.copy_(x_all)
            np.copyto(plan.idx_host.numpy(), order, casting="unsafe")      # pinned staging: async H2D
            plan.idx.copy_(plan.idx_host, non_blocking=True)
            plan.run()
            plan.out_host.copy_(plan.out, non_blocking=True)
            plan.fetch_overflow()
            torch.cuda.current_stream().synchronize()
            if not plan.overflowed():
                self._last_raw = plan.out_host.numpy()
                return self._last_raw[3].copy()
            # some candidate list was empty or overflowed (heavy ties): the replayed graph carries no exhaustive-scan
            # launches, so this call is repeated eagerly below, which does
            plan.clear_overflow()
        idx = torch.from_numpy(order.astype(np.int32)).to(eng.dev, non_blocking=True)
        q_class = torch.from_numpy(labels[order].astype(np.int32)).to(eng.dev, non_blocking=True)
        out = torch.empty((4, n_total), dtype=torch.float64, device=eng.dev)
        if promoted:
            self._call_promoted(x_all, idx, q_class, q_off, out)
        else:
            E.dsa_scores(eng, x_all, idx, q_class, q_off, out, comm, self.use_filter)
        self._last_raw = out.cpu().numpy()
        return self._last_raw[3].copy()

    def _prepare(self, activations, predictions):
        """The checks and the upload every call shares.  Returns the test traces in the engine's landing buffer (in the
        scoring dtype), the class-grouped order and offsets of the rows to score, the labels, and whether the call
        is promoted (float64 test traces against float32 training traces)."""
        import torch

        from .. import engine as E

        labels = _class_predictions(E.host_array(predictions))
        dev_ats = E.device_matrix(activations)        # traces already in HBM: no host round trip
        host_ats = _flatten_layers(activations) if dev_ats is None else None
        # NumPy promotes `from_ats[:, None] - to_ats` (surprise.py:638): float64 test traces against float32
        # training traces are scored in float64 (the training traces widened exactly)
        wide = (dev_ats.dtype == torch.float64) if dev_ats is not None else \
            (np.result_type(host_ats.dtype, self._compute_dtype) == np.float64)
        compute = np.dtype(np.float64) if wide else self._compute_dtype
        promoted = compute != self._compute_dtype
        if promoted and self._comm is not None and self._comm.world > 1:
            raise TypeError("N_train-sharded DSA scores in the dtype of the training traces "
                            f"({self._compute_dtype}); got float64 test traces")
        torch_dtype = torch.float64 if compute == np.float64 else torch.float32
        if dev_ats is not None:
            target_ats = dev_ats.to(torch_dtype)
        else:
            target_ats = host_ats if host_ats.dtype == compute else host_ats.astype(compute)
        eng = self._engine
        if target_ats.ndim != 2 or int(target_ats.shape[1]) != eng.d:
            # the reference's `from_ats[:, None] - to_ats` raises the same kind of error (surprise.py:638)
            raise ValueError(f"operands could not be broadcast together: test traces have shape "
                             f"{tuple(target_ats.shape)}, training traces have {eng.d} features")
        n_total = labels.shape[0]
        # start the (asynchronous, if the caller's buffer is pinned) upload first; the host-side
        # planning below overlaps with it
        x_all = None
        if n_total:
            x_all = eng.input_buffer(n_total, torch_dtype)
            x_all.copy_(target_ats if dev_ats is not None else torch.from_numpy(np.ascontiguousarray(target_ats)),
                        non_blocking=True)
        # class-grouped order; rows labelled >= num_classes are never scored by the reference
        # (its result buffer is np.empty there, surprise.py:576-580) -> NaN here.
        order, q_off = E.class_layout(labels, int(self.num_classes))
        for c in range(int(self.num_classes)):
            if q_off[c + 1] > q_off[c] and len(self.class_matrix[c]) in (0, self.train_predictions.shape[0]):
                raise ValueError("zero-size array to reduction operation minimum which has no identity")
        self._last_dtype = compute
        return x_all, order, q_off, labels, promoted

    def _call_promoted(self, x_all, idx, q_class, q_off, out):
        """float64 test traces against float32 training traces, exactly as NumPy promotes them in the reference:
        stage 1 (`from_ats[:, None] - to_ats`, surprise.py:638) runs in float64 on the exactly widened training traces
        (a float64 twin of the engine, built on first use); stage 2's operands are both float32 TRAINING rows, so it
        stays float32 (surprise.py:627-629); dsa = dist_a (f64) / dist_b (f32 -> f64).  Eager launches."""
        import torch

        from .. import _lib
        from .. import engine as E

        if self._engine_wide is None:
            train = self.train_activations
            train = train.to(torch.float64) if isinstance(train, torch.Tensor) else np.asarray(train, dtype=np.float64)
            self._engine_wide = E.NnEngine.from_host(train, self.train_predictions, int(self.num_classes),
                                                     np.arange(train.shape[0]), seeds=False)
        eng, wide = self._engine, self._engine_wide
        dist_a, pos, gid, _ = wide.search(x_all, q_class, q_off, _lib.RANGE_SAME_CLASS, self.use_filter, q_idx=idx)
        winners = eng.gather(pos)                      # float32 training rows (same class-sorted positions)
        dist_b = eng.search(winners, q_class, q_off, _lib.RANGE_OTHER_CLASSES, self.use_filter)[0]
        E.reset_unscored(out, idx.shape[0])
        E.pack_out(dist_a, dist_b.to(torch.float64), gid, idx, out)

    # Results of the most recent call (exact widenings of the device values; valid until the next call)
    @property
    def last_dist_a(self) -> np.ndarray:
        return self._last_raw[0].astype(self._last_dtype or self._compute_dtype)

    @property
    def last_dist_b(self) -> np.ndarray:
        return self._last_raw[1].astype(self._last_dtype or self._compute_dtype)

    @property
    def last_winner_index(self) -> np.ndarray:
        return self._last_raw[2].astype(np.int64)
