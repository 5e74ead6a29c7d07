"""Gaussian KDE with the reference's covariance "stabilisation", evaluated on the GPU.

Mirror of `/root/reference/src/core/stable_kde.py` (a subclass of scipy==1.4.1's
`gaussian_kde`).  The fit is the reference's float64 host arithmetic, restated line by line:
Scott factor n^(-1/(d+4)); `np.cov(bias=False, aweights=1/n)`; while any eigenvalue of
cov*factor^2 is <= 0 REPLACE the diagonal by 1e-10 * 2^k, giving up past 1e-5
(`prepare_failed` -> every density 0, stable_kde.py:55-77,99-100); inverse; Cholesky of
2*pi*covariance (raises LinAlgError like the reference when not positive definite).

evaluate() is scipy 1.4.1's `gaussian_kernel_estimate`:
    density_j = (1/n) * (2 pi)^(-d/2) * prod(diag(W)) * sum_i exp(-|p_i - q_j|^2 / 2),
    W = cholesky(inv_cov), p = data . W, q = x . W
computed by libb200tip.so in the log domain (split-bf16 tensor-core dot products, fused
online log-sum-exp) and converted back to a float64 density here, so underflow to exactly 0
(-> LSA = +inf, surprise.py:495) happens where the reference's float64 sum underflows.
"""
from __future__ import annotations

import math
import warnings
from typing import Optional

import numpy as np


class StableGaussianKDE:
    MAX_INCREMENT = 1e-5

    def __init__(self, dataset, bw_method=None, weights=None, source_columns: Optional[np.ndarray] = None,
                 comm=None):
        if bw_method is not None or weights is not None:
            raise NotImplementedError("only the reference's usage (scott bandwidth, uniform weights) is supported")
        self.dataset = np.atleast_2d(np.asarray(dataset)).astype(np.float64)     # stable_kde.py:22
        if not self.dataset.size > 1:
            raise ValueError("`dataset` input should have multiple elements.")
        self.d, self.n = self.dataset.shape
        self.weights = np.ones(self.n) / self.n
        self.neff = 1.0 / np.sum(self.weights ** 2)
        self.source_columns = None if source_columns is None else np.asarray(source_columns, dtype=np.int32)
        self._engine = None
        self._comm = comm          # N_train-sharded evaluation (engine.TrainShardComm); the fit is replicated
        self._compute_covariance()
        if not self.prepare_failed:
            self._upload()

    def scotts_factor(self):
        return np.power(self.neff, -1.0 / (self.d + 4))

    covariance_factor = scotts_factor

    # -- fit (host, float64) ---------------------------------------------------------------
    def _compute_covariance(self):
        self.factor = self.covariance_factor()
        cov = np.atleast_2d(np.cov(self.dataset, rowvar=1, bias=False, aweights=self.weights))
        cov = self._stabilize_covariance(cov)
        if self.prepare_failed:
            self._data_inv_cov = None
            return
        self._data_covariance = cov
        try:
            self._data_inv_cov = np.linalg.inv(cov)
        except np.linalg.LinAlgError:
            self.prepare_failed = True
            self._data_inv_cov = None
            return
        self.covariance = cov * self.factor ** 2
        self.inv_cov = self._data_inv_cov / self.factor ** 2
        chol = np.linalg.cholesky(self.covariance * 2 * np.pi)
        self.log_det = 2 * np.log(np.diag(chol)).sum()
        self._norm_factor = np.sqrt(np.linalg.det(2 * np.pi * self.covariance))

    def _stabilize_covariance(self, covariance):
        increment = 1e-10
        while np.any(np.linalg.eigh(covariance * self.factor ** 2)[0] <= 0):
            np.fill_diagonal(covariance, increment)
            if increment > self.MAX_INCREMENT:
                warnings.warn("Was not able to fix numerical imprecision in covariance matrix."
                              "Failing silently. All likelihoods will be reported as 0.")
                self.prepare_failed = True
                return None
            increment += increment
        self.prepare_failed = False
        return covariance

    @classmethod
    def from_device(cls, x, cols: Optional[np.ndarray] = None, mean=None, timing: Optional[dict] = None
                    ) -> "StableGaussianKDE":
        """StableGaussianKDE(x[:, cols].T) fitted on the GPU (engine.kde_fit, float64): x is an [n, D] float32 /
        float64 device matrix, cols the kept source columns (None: all of them), mean x's float64 column mean
        (engine.col_var's, optional).  Same attributes and errors as the host fit; dataset, covariance, inv_cov,
        whitening, _data_covariance, _data_inv_cov and mean are held on the device and copied to the host on first
        access.  The training operand is the fit's own fp32 (x[:, cols] - mean) @ W, which never leaves the GPU."""
        import torch

        from .. import engine as E

        n, width = int(x.shape[0]), int(x.shape[1])
        d = width if cols is None else len(cols)
        if not n * d > 1:
            raise ValueError("`dataset` input should have multiple elements.")
        self = cls.__new__(cls)
        self.d, self.n = d, n
        self.weights = np.ones(self.n) / self.n
        self.neff = 1.0 / np.sum(self.weights ** 2)
        self.source_columns = None if cols is None else np.asarray(cols, dtype=np.int32)
        self._engine, self._comm = None, None
        fit = E.kde_fit(x, cols, mean, timing)
        self.factor = fit["factor"]
        self.prepare_failed = fit["prepare_failed"]
        rows = fit["rows"]
        f2 = self.factor ** 2
        self._lazy = {"dataset": lambda: rows.t().to(torch.float64), "mean": lambda: fit["mean"]}
        if "covariance" not in fit:                  # failed fit: the host keeps no inverse either
            self._data_inv_cov = None
            return self
        self._lazy.update({"_data_covariance": lambda: fit["covariance"], "_data_inv_cov": lambda: fit["inv"],
                           "covariance": lambda: fit["covariance"] * f2, "inv_cov": lambda: fit["inv"] / f2,
                           "whitening": lambda: fit["whitening"]})
        self.log_det = fit["log_det"]
        self._norm_factor = fit["norm_factor"]
        self._attach(fit["diag_w"], fit["p"], fit["whitening"].to(torch.float32), fit["mean"])
        return self

    def __getattr__(self, name):
        """device-held attributes of a from_device fit, copied to the host on first access"""
        lazy = self.__dict__.get("_lazy")
        if lazy is None or name not in lazy:
            raise AttributeError(f"{type(self).__name__!r} object has no attribute {name!r}")
        value = lazy.pop(name)().cpu().numpy()
        setattr(self, name, value)
        return value

    # -- device state ----------------------------------------------------------------------
    def _upload(self):
        import torch

        self.whitening = np.linalg.cholesky(self.inv_cov)                 # scipy 1.4.1: cholesky(precision)
        self.mean = self.dataset.mean(axis=1)
        # squared distances are translation invariant: centre before whitening so the split-bf16
        # operands carry the spread, not the offset, of the traces
        p = (self.dataset.T - self.mean) @ self.whitening
        self._attach(np.diag(self.whitening), p, torch.from_numpy(self.whitening.astype(np.float32)),
                     torch.from_numpy(self.mean))

    def _attach(self, diag_w: np.ndarray, p, w32, mu):
        """norm / log_norm from the whitening factor's diagonal, the KDE engine over the training operand p, and the
        query whitening's device operands (w32 fp32 [d, d], mu float64 [d])."""
        import torch

        from .. import engine as E

        norm = math.pow(2 * math.pi, -self.d / 2.0)
        for i in range(self.d):
            norm *= diag_w[i]
        self.norm = norm
        self.log_norm = -self.d / 2.0 * math.log(2 * math.pi) + float(np.sum(np.log(diag_w)))
        self._engine = E.KdeEngine(p, self._comm)
        dev = self._engine.dev
        self._w_dev = w32.to(dev)
        self._mu_dev = mu.to(dev)
        self._cols_dev = None if self.source_columns is None else torch.from_numpy(self.source_columns).to(dev)
        self._plans = E.BoundedCache(4)
        self._seen_shapes = E.BoundedCache(65)
        self._pinned_pool = E.BoundedCache(33)

    # -- score -----------------------------------------------------------------------------
    def evaluate(self, points) -> np.ndarray:
        """scipy convention: points is (d, m) (or (d,) for one point)."""
        points = np.atleast_2d(np.asarray(points))
        d, m = points.shape
        if d != self.d:
            if d == 1 and m == self.d:
                points = np.reshape(points, (self.d, 1))
                m = 1
            else:
                raise ValueError(f"points have dimension {d}, dataset has dimension {self.d}")
        if self.prepare_failed:
            return np.zeros(m)
        return self._density(np.ascontiguousarray(points.T), preselected=True)

    __call__ = evaluate

    def evaluate_rows(self, rows: np.ndarray) -> np.ndarray:
        """rows: (m, all source columns); the kept columns are gathered on the GPU."""
        return self.evaluate_rows_begin(rows).finish()

    def evaluate_rows_begin(self, rows):
        if self.prepare_failed:
            return _PendingDensity(self, None, -int(rows.shape[0]), 0, None, None)
        return self._density_begin(rows, preselected=self.source_columns is None)

    # Fast pass (one fp16 segment) is accepted when, on a sample of the queries, its -log density agrees with the
    # three-segment pass to 4e-5 relative.  The error is measured on the data at hand, not assumed from a model:
    # per-input errors are zero-mean rounding noise (the dominant kernel term's 2^-12 relative operand rounding), so
    # the largest of 128 samples sits near 2.5 sigma and the largest of 1e4..1e5 inputs near 4..4.4 sigma — at most
    # 1.8x the sample maximum, i.e. <= 7.2e-5 < north_star's rtol 1e-4.  One failed check retires the fast pass for
    # this KDE.  (C3: 2.8e-5 on the sample, 3.2e-5 worst of 256 other inputs against the float64 restatement of scipy.)
    FAST_MIN_ROWS = 1024
    FAST_SAMPLE = 128
    FAST_RTOL = 4e-5

    def _density(self, rows: np.ndarray, preselected: bool) -> np.ndarray:
        return self._density_begin(rows, preselected).finish()

    def _density_begin(self, rows, preselected: bool) -> "_PendingDensity":
        """Launches everything a density evaluation needs and starts the device->host copy of its partials into
        pinned memory WITHOUT synchronising; `finish()` waits for that copy and does the float64 host math (and,
        if the fast pass fails its check, the three-segment re-run).  Lets `MultiModalSA` keep the per-class KDEs of
        a batch in flight together (handler_surprise.py:26: one LSA per class)."""
        import torch

        from .. import engine as E

        eng = self._engine
        if isinstance(rows, torch.Tensor):            # device-resident traces
            if rows.dtype not in (torch.float32, torch.float64):
                rows = rows.to(torch.float32)
        elif rows.dtype not in (np.float32, np.float64):
            rows = rows.astype(np.float64)
        m = rows.shape[0]
        if m == 0:
            return _PendingDensity(self, None, 0, 0, None, None)
        fast = bool(eng.fast_ok and m >= self.FAST_MIN_ROWS)
        self.last_operands = "split-bf16 x3"
        # A batch shape seen for the second time is captured as ONE CUDA graph (whiten -> pack -> wgmma log-sum-exp ->
        # merge, plus the sampled three-segment pass of the fast check) and replayed from then on: the ~20 small
        # launches of a call are otherwise issued more slowly by the host than the GPU executes them (per-class LSA:
        # ten such chains per scoring call, handler_surprise.py:26).
        dt = (torch.float64 if rows.dtype in (torch.float64, np.float64) else torch.float32)
        key = (int(m), int(rows.shape[1]), dt, bool(preselected), fast)
        plan = self._plans.get(key)
        if plan is None and self._seen_shapes.touch(key) and E.GRAPHS and eng.comm is None:
            plan = self._plans.get_or_make(key, lambda: _DensityPlan(self, key))
        if plan is not None:
            src = rows if isinstance(rows, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(rows))
            plan.x_in.copy_(src, non_blocking=True)
            plan.graph.replay()
            packed, n_s, q = plan.packed, plan.n_s, plan.q
        else:
            packed, n_s, q = self._density_body(E.to_device(rows, eng.dev), preselected, fast)
        host = self._pinned(packed.shape)
        host.copy_(packed, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        return _PendingDensity(self, host, m, n_s, done, q if fast else None)

    def _density_body(self, x, preselected: bool, fast: bool):
        """device work of one density evaluation: (packed partials [2, m (+ 2 n_s)] float64, n_s, whitened queries)"""
        import torch

        from .. import engine as E

        eng = self._engine
        m = x.shape[0]
        E.keep_for_capture(self._cols_dev, self._mu_dev, self._w_dev)
        q = E.whiten(x, None if preselected else self._cols_dev, self._mu_dev, self._w_dev)
        if fast:
            eng.flags.zero_()
            mx, sm, qsq = eng.log_kernel_sum(q, fast=True)
            sel = torch.arange(0, m, max(1, m // self.FAST_SAMPLE), device=eng.dev)[:self.FAST_SAMPLE]
            mx3, sm3, qsq3 = eng.log_kernel_sum(q.index_select(0, sel).contiguous())
            packed = torch.cat([torch.stack([mx.to(torch.float64) - 0.5 * qsq.to(torch.float64), sm.to(torch.float64)]),
                                torch.stack([mx3.to(torch.float64) - 0.5 * qsq3.to(torch.float64), sm3.to(torch.float64)]),
                                torch.stack([sel.to(torch.float64), eng.flags.to(torch.float64).expand(sel.shape[0])])],
                               dim=1)
            return packed, int(sel.shape[0]), q
        mx, sm, qsq = eng.log_kernel_sum(q)
        packed = torch.stack([mx.to(torch.float64) - 0.5 * qsq.to(torch.float64), sm.to(torch.float64)])
        return packed, 0, q

    def _pinned(self, shape):
        """pinned landing buffers, recycled per shape (cudaHostAlloc is slow)"""
        import torch

        key = tuple(shape)
        return self._pinned_pool.get_or_make(key, lambda: torch.empty(key, dtype=torch.float64, pin_memory=True))

    def _finish(self, log_max: np.ndarray, rel_sum: np.ndarray) -> np.ndarray:
        """float64 density from the log-domain partials, with the reference's underflow:
        in gaussian_kernel_estimate every term is fl(fl(exp(-arg/2)*norm)*w); if the largest
        term is 0 all are, and the density is exactly 0."""
        weight = 1.0 / self.n
        with np.errstate(under="ignore", divide="ignore", invalid="ignore"):
            log_density = self.log_norm + math.log(weight) + log_max + np.log(rel_sum)
            density = np.exp(log_density)
            largest_term = (np.exp(log_max) * self.norm) * weight
        density[largest_term == 0] = 0.0
        density[~np.isfinite(log_max)] = 0.0
        return density


class _DensityPlan:
    """One density evaluation of a fixed batch shape as a CUDA graph (see StableGaussianKDE._density_begin)."""

    def __init__(self, kde, key):
        import torch

        from .. import engine as E

        m, d_in, dt, preselected, fast = key
        dev = kde._engine.dev
        self.x_in = torch.zeros((m, d_in), dtype=dt, device=dev)

        def body():
            self.packed, self.n_s, self.q = kde._density_body(self.x_in, preselected, fast)

        _, (self.graph,), self._keep_alive = E.capture_graphs([(body, True)], dev)


class _PendingDensity:
    """A density evaluation in flight (see StableGaussianKDE._density_begin)."""

    def __init__(self, kde, host, m, n_s, done, q):
        self.kde, self.host, self.m, self.n_s, self.done, self.q = kde, host, m, n_s, done, q

    def finish(self) -> np.ndarray:
        import torch

        kde = self.kde
        if self.m <= 0:
            return np.zeros(-self.m)               # empty batch, or a KDE whose fit failed: all densities 0
        self.done.synchronize()
        packed = self.host.numpy().copy()
        m, n_s = self.m, self.n_s
        if n_s == 0:
            return kde._finish(packed[0], packed[1])
        fast_lm, fast_rs = packed[0, :m], packed[1, :m]
        ref_lm, ref_rs = packed[0, m:m + n_s], packed[1, m:m + n_s]
        idx = packed[0, m + n_s:].astype(np.int64)
        overflow = packed[1, m + n_s] != 0
        with np.errstate(divide="ignore", invalid="ignore", under="ignore"):
            l_fast = -(kde.log_norm - math.log(kde.n) + fast_lm[idx] + np.log(fast_rs[idx]))
            l_ref = -(kde.log_norm - math.log(kde.n) + ref_lm + np.log(ref_rs))
            both = np.isfinite(l_fast) & np.isfinite(l_ref)
            worst = float(np.max(np.abs(l_fast[both] - l_ref[both]) / np.abs(l_ref[both]))) if both.any() else 0.0
        same_inf = np.array_equal(np.isfinite(l_fast), np.isfinite(l_ref))
        kde.last_fast_check = {"rows": int(n_s), "max_rel_diff": worst,
                               "accepted": bool(not overflow and same_inf and worst <= kde.FAST_RTOL)}
        if kde.last_fast_check["accepted"]:
            kde.last_operands = "fp16 x1 (verified on %d sampled rows: max rel diff %.2e)" % (n_s, worst)
            # (the sampled rows keep their fast values too: a row's score must not depend on where it sits in the batch)
            return kde._finish(fast_lm, fast_rs)
        eng = kde._engine
        eng.fast_ok = False
        mx, sm, qsq = eng.log_kernel_sum(self.q)
        mx = mx.to(torch.float64) - 0.5 * qsq.to(torch.float64)
        out = torch.stack([mx, sm.to(torch.float64)]).cpu().numpy()
        return kde._finish(out[0], out[1])
