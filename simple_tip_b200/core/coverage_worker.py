"""The study's neuron-coverage arm for PyTorch models (handler_coverage.py:20-132, `CoverageWorker`).

Walks the training set once for the per-neuron min / max / std (`AggregateStatisticsCollector`), builds the twelve
coverage metrics of the study, then scores every test set and orders it by CAM, timing each phase as the reference
does.  The traces come from forward hooks (`activations.TransparentModel`) and stay in HBM: every metric's profile is
written bit-packed by its own kernel (`packed()`) and ordered by `prioritizers.cam_from_bits`; no profile leaves the
device and nothing is written to disk.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

from .activations import HookedModelHandler, TransparentModel
from .aggregate_statistics import AggregateStatisticsCollector
from .neuron_coverage import KMNC, NAC, NBC, SNAC, TKNC, CoverageMethod, _score_dtype
from .prioritizers import cam_from_bits
from .timer import Timer


class CoverageWorker(HookedModelHandler):
    """`CoverageWorker(base_model, training_set)` + `evaluate_all(test_dataset, test_dataset_id)` of
    handler_coverage.py for a `torch.nn.Module`.

    nc_layers: as `TransparentModel`'s activation_layers (child indices or dotted submodule names); the model's own
    output is not a coverage layer.  training_data / test data: a tensor or an array [N, ...], run through the model
    in badges of `batch_size` on the model's device.  Every timer ends with a synchronise of the current CUDA device
    (and the model's, when that is another one), so device work is inside the phase that launched it.

    Writing the reference's result files (eval_prioritization.py:174-193; `prioritization.evaluate` runs the whole
    experiment, this arm included):

        worker = CoverageWorker(model, [1, 2, 4, 5], x_train)
        for ds_name, x in {"nominal": x_test, "ood": x_ood}.items():
            times, scores, orders = worker.evaluate_all(x)
            for metric in worker.metrics:
                results.persist_tip(out, case_study, ds_name, model_id, metric, scores[metric], orders[metric],
                                    times[metric])
    """

    def __init__(self, model, nc_layers: Sequence, training_data, batch_size: int = 128):
        self.nc_layers = list(nc_layers)
        self.base_model = TransparentModel(model, self.nc_layers, include_last_layer=False)
        self.batch_size = batch_size
        self.metrics: Dict[str, CoverageMethod] = {}
        self.setup_times: Dict[str, float] = {}

        x = self._inputs(training_data, "training_data")
        agg_stats = AggregateStatisticsCollector()
        pred_timer = Timer()
        for start in range(0, x.shape[0], batch_size):           # handler_coverage.py:33-42
            badge = x[start:start + batch_size]
            activations = self._synced(lambda: self.base_model.get_activations(badge), pred_timer)
            agg_stats.track(activations)
        mins, maxs, std = agg_stats.get()
        self.mins, self.maxs, self.stds = mins, maxs, std          # per layer, layer-shaped

        # handler_coverage.py:49-101; the collector books min, max and Welford on its welford timer
        nbc_debit = agg_stats.min_timer.get() + agg_stats.max_timer.get() + pred_timer.get() + agg_stats.welford_timer.get()
        for s in (0, 0.5, 1):
            self._add_metric(f"NBC_{s}", lambda s=s: NBC(mins=mins, maxs=maxs, stds=std, scaler=s), nbc_debit)
        snac_debit = agg_stats.welford_timer.get() + agg_stats.max_timer.get() + pred_timer.get()
        for s in (0, 0.5, 1):
            self._add_metric(f"SNAC_{s}", lambda s=s: SNAC(maxs=maxs, stds=std, scaler=s), snac_debit)
        self._add_metric("NAC_0", lambda: NAC(cov_threshold=0.0))
        self._add_metric("NAC_0.75", lambda: NAC(cov_threshold=0.75))
        for k in (1, 2, 3):
            self._add_metric(f"TKNC_{k}", lambda k=k: TKNC(top_neurons=k))
        kmnc_debit = agg_stats.min_timer.get() + agg_stats.max_timer.get() + pred_timer.get()
        self._add_metric("KMNC_2", lambda: KMNC(mins, maxs, sections=2), kmnc_debit)

    def _inputs(self, data, what: str):
        """data as a tensor on the model's device; ValueError for an empty set"""
        import torch

        x = data if isinstance(data, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(data))
        if x.shape[0] == 0:
            raise ValueError(f"{what} holds no inputs")
        return x.to(self._model_device())

    def _add_metric(self, metric_id: str, metric_supplier: Callable[[], CoverageMethod], time_debit: float = 0.0):
        timer = Timer()
        self.metrics[metric_id] = self._synced(metric_supplier, timer)
        self.setup_times[metric_id] = time_debit + timer.get()

    def _traces(self, data) -> Tuple[List, object]:
        """The test set's hooked layers on the scoring device (moved there once if the model lives elsewhere), and
        the same traces flattened to one [N, D] matrix, in input order."""
        import torch

        from .. import engine as E

        dev = E.require_cuda()
        layers = [a.to(dev) for a in self.base_model.collect(self._inputs(data, "test data"), self.batch_size)]
        flat = torch.cat([a.reshape(a.shape[0], -1) for a in layers], dim=1)
        return layers, flat

    @staticmethod
    def _cam_sanity_check(cam_order, scores):
        assert len(cam_order) == len(set(cam_order)) == scores.shape[0], "CAM order is not unique or not complete"

    def evaluate_all(self, test_dataset, test_dataset_id=None
                     ) -> Tuple[Dict[str, List[float]], Dict[str, np.ndarray], Dict[str, np.ndarray]]:
        """(times, all_scores, cam_orders), each keyed by metric name (handler_coverage.py:103-132).

        times[m] = [setup, pred, quant, cam] in seconds: setup = the metric's debit of the training walk plus its
        construction; pred = collecting and flattening the test set's traces (once, shared by every metric, as the
        reference adds up its per-badge walk for each metric); quant = `metric.packed(...)` with the scores' download;
        cam = `cam_from_bits` on the packed profile.  all_scores[m]: NumPy, in the dtype the reference's `sum_score`
        picks; cam_orders[m]: int64.  Rows are in input order.  test_dataset_id is accepted for the reference's
        signature; nothing is written anywhere.  An empty test set raises ValueError before any launch."""
        from .. import _lib

        pred_timer = Timer()
        layers, flat = self._synced(lambda: self._traces(test_dataset), pred_timer)
        d = int(flat.shape[1])
        words = int(_lib.load().tip_cover_packed_words(d))
        times, all_scores, cam_orders = {}, {}, {}
        for metric_id, metric in self.metrics.items():
            quant_timer = Timer()

            def quant():
                score, bits = metric.packed(layers if isinstance(metric, TKNC) else flat)
                # sum_score's dtype: from the dense profile's entries per sample, d x planes
                return score.cpu().numpy().astype(_score_dtype(d * (int(bits.shape[1]) // words))), bits
            scores, bits = self._synced(quant, quant_timer)
            cam_timer = Timer()
            order = self._synced(lambda: np.array(list(cam_from_bits(scores, bits)), dtype=np.int64), cam_timer)
            self._cam_sanity_check(order, scores)
            del bits
            times[metric_id] = [self.setup_times[metric_id], pred_timer.get(), quant_timer.get(), cam_timer.get()]
            all_scores[metric_id] = scores
            cam_orders[metric_id] = order
        return times, all_scores, cam_orders
