"""The study's neuron-coverage arm for PyTorch models (handler_coverage.py:20-132, `CoverageWorker`).

Walks the training set once for the per-neuron min / max / std (`AggregateStatisticsCollector`), builds the twelve
coverage metrics of the study, then scores every test set and orders it by CAM, timing each phase as the reference
does.  The traces come from forward hooks (`activations.TransparentModel`) and stay in HBM: every metric's profile is
written bit-packed by its own kernel (`packed()`) and ordered by `prioritizers.cam_from_bits`; no profile leaves the
device and nothing is written to disk.
"""
from __future__ import annotations

import functools
import math
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import prioritizers as P
from .activations import HookedModelHandler, TransparentModel
from .aggregate_statistics import AggregateStatisticsCollector
from .neuron_coverage import KMNC, NAC, NBC, SNAC, TKNC, CoverageMethod, _score_dtype
from .timer import Timer

# The study's twelve coverage metrics (handler_coverage.py:49-101) as (id, debit, factory): the factory builds the
# metric from one model's per-layer mins, maxs and stds, and the debit names its share of the training walk
# (`_walk_debits`).  A debit of None marks a metric built from no training statistics: it is charged nothing and
# holds no state, so one object serves every model of a stack.
METRICS = (
    [(f"NBC_{s}", "NBC", lambda mn, mx, sd, s=s: NBC(mins=mn, maxs=mx, stds=sd, scaler=s)) for s in (0, 0.5, 1)]
    + [(f"SNAC_{s}", "SNAC", lambda mn, mx, sd, s=s: SNAC(maxs=mx, stds=sd, scaler=s)) for s in (0, 0.5, 1)]
    + [("NAC_0", None, lambda *_: NAC(cov_threshold=0.0)), ("NAC_0.75", None, lambda *_: NAC(cov_threshold=0.75))]
    + [(f"TKNC_{k}", None, lambda *_, k=k: TKNC(top_neurons=k)) for k in (1, 2, 3)]
    + [("KMNC_2", "KMNC", lambda mn, mx, sd: KMNC(mn, mx, sections=2))])


def _walk_debits(agg_stats: AggregateStatisticsCollector, pred_timer: Timer) -> Dict:
    """The debits of `METRICS` in seconds; the collector books min, max and Welford on its welford timer."""
    mn, mx, wf = agg_stats.min_timer.get(), agg_stats.max_timer.get(), agg_stats.welford_timer.get()
    pred = pred_timer.get()
    return {"NBC": mn + mx + pred + wf, "SNAC": wf + mx + pred, "KMNC": mn + mx + pred, None: 0.0}


class _CoverageArm(HookedModelHandler):
    """What `CoverageWorker` and `StackedCoverageWorker` share: the coverage arm of the M models hooked in
    `self.base_model`, all fed the same inputs.  A subclass sets `models`, `base_model` and `batch_size` and gives
    `_activations(badge)`, every hooked layer of one forward on the badge as [M, b, *layer shape], and
    `_cam(scores, bits)`, the M CAM orders of M profiles."""

    models = 1

    def _walk(self, training_data):
        """The training walk (handler_coverage.py:33-42) and the metrics of `METRICS`.  Every hooked output goes to one
        `AggregateStatisticsCollector` as rows [b, M, *layer shape], so one `tip_stats_update` per layer and badge
        serves all M models.  Sets `self._metrics` (per metric, one object per model, or one for all M models when
        the metric holds no state) and `self.setup_times` (split evenly over the M models); returns (mins, maxs,
        stds), each per model a list of layer-shaped arrays."""
        x = self._inputs(training_data, "training_data")
        agg_stats = AggregateStatisticsCollector()
        pred_timer = Timer()
        for start in range(0, x.shape[0], self.batch_size):
            activations = self._synced(lambda: self._activations(x[start:start + self.batch_size]), pred_timer)
            agg_stats.track([a.transpose(0, 1) for a in activations])     # [b, M, *layer shape]
        mins, maxs, stds = ([[layer[m] for layer in stat] for m in range(self.models)] for stat in agg_stats.get())

        debits = _walk_debits(agg_stats, pred_timer)
        self._metrics: Dict[str, List[CoverageMethod]] = {}
        self.setup_times: Dict[str, float] = {}
        for metric_id, debit, factory in METRICS:
            timer = Timer()
            built = range(1 if debit is None else self.models)
            self._metrics[metric_id] = self._synced(lambda: [factory(mins[m], maxs[m], stds[m]) for m in built], timer)
            self.setup_times[metric_id] = (debits[debit] + timer.get()) / self.models
        return mins, maxs, stds

    def _traces(self, data):
        """The test set's traces as one model-major [M, N, D] tensor on the scoring device (each model's layers
        flattened and concatenated in layer order, in the dtype `torch.cat` of the layers gives), and each layer's
        shape."""
        import torch

        from .. import engine as E

        dev = E.require_cuda()
        x = self._inputs(data, "test data")
        n = int(x.shape[0])
        flat, shapes = None, None
        for start in range(0, n, self.batch_size):
            acts = self._activations(x[start:start + self.batch_size])
            if flat is None:
                shapes = [tuple(a.shape[2:]) for a in acts]
                dtype = functools.reduce(torch.promote_types, [a.dtype for a in acts])
                flat = torch.empty((self.models, n, sum(math.prod(s) for s in shapes)), dtype=dtype, device=dev)
            off = 0
            for a in acts:
                a = a.reshape(a.shape[0], a.shape[1], -1)
                flat[:, start:start + a.shape[1], off:off + a.shape[2]].copy_(a)
                off += a.shape[2]
        return flat, shapes

    def _model_major(self, data):
        """What `_evaluate` scores: `_traces`' [M, N, D] tensor and layer shapes."""
        return self._traces(data)

    @staticmethod
    def _cam_sanity_check(cam_order, scores):
        assert len(cam_order) == len(set(cam_order)) == scores.shape[0], "CAM order is not unique or not complete"

    def _evaluate(self, test_dataset
                  ) -> List[Tuple[Dict[str, List[float]], Dict[str, np.ndarray], Dict[str, np.ndarray]]]:
        """M (times, all_scores, cam_orders) triples in `CoverageWorker.evaluate_all`'s form, each phase's time split
        evenly over the M models.  NAC runs once on the traces' [M * N, D] view, NBC, SNAC and KMNC on each model's
        [N, D] slice, TKNC on each model's layer views."""
        import torch

        from .. import _lib

        models = self.models
        pred_timer = Timer()
        flat, shapes = self._synced(lambda: self._model_major(test_dataset), pred_timer)
        n, d = int(flat.shape[1]), int(flat.shape[2])
        widths = [math.prod(s) for s in shapes]
        words = int(_lib.load().tip_cover_packed_words(d))
        results = [({}, {}, {}) for _ in range(models)]
        copies = {}

        def layers(m):
            """model m's layers as contiguous [N, w] copies (`tip_tknc` reads contiguous rows), kept for the next TKNC
            metric; one model's copies at a time"""
            if m not in copies:
                copies.clear()
                copies[m] = [t.contiguous() for t in flat[m].split(widths, dim=1)]
            return copies[m]

        for metric_id, metric in self._metrics.items():
            if not isinstance(metric[0], TKNC):
                copies.clear()
            quant_timer = Timer()

            def quant():
                if isinstance(metric[0], NAC):                  # one launch over the [M * N, D] view
                    score, bits = metric[0].packed(flat.view(models * n, d))
                    score, bits = score.view(models, n), bits.view(models, n, -1)
                else:
                    score, bits = None, None
                    for m in range(models):
                        if isinstance(metric[0], TKNC):
                            s, b = metric[0].packed(layers(m))
                        else:
                            s, b = metric[m].packed(flat[m])
                        if models == 1:                         # one model's profile is taken as it is
                            score, bits = s[None], b[None]
                            continue
                        if bits is None:
                            score = torch.empty((models, n), dtype=s.dtype, device=s.device)
                            bits = torch.empty((models, n, int(b.shape[1])), dtype=b.dtype, device=b.device)
                        score[m].copy_(s)
                        bits[m].copy_(b)
                        del s, b
                # sum_score's dtype: from the dense profile's entries per sample, d x planes
                return score.cpu().numpy().astype(_score_dtype(d * (int(bits.shape[2]) // words))), bits
            scores, bits = self._synced(quant, quant_timer)
            cam_timer = Timer()
            orders = self._synced(lambda: self._cam(scores, bits), cam_timer)
            del bits
            for m, order in enumerate(orders):
                self._cam_sanity_check(order, scores[m])
                times, all_scores, cam_orders = results[m]
                times[metric_id] = [self.setup_times[metric_id], pred_timer.get() / models, quant_timer.get() / models,
                                    cam_timer.get() / models]
                all_scores[metric_id] = scores[m]
                cam_orders[metric_id] = order
        return results


class CoverageWorker(_CoverageArm):
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
        (self.mins,), (self.maxs,), (self.stds,) = self._walk(training_data)     # per layer, layer-shaped
        self.metrics: Dict[str, CoverageMethod] = {metric_id: m[0] for metric_id, m in self._metrics.items()}

    def _activations(self, badge):
        return [a[None] for a in self.base_model.get_activations(badge)]

    def _traces(self, data):
        """The test set's hooked layers on the scoring device, and the same traces flattened to one [N, D] matrix, in
        input order; the layers are views of the matrix."""
        flat, shapes = super()._traces(data)
        flat = flat[0]
        layers, off = [], 0
        for shape in shapes:
            width = math.prod(shape)
            layers.append(flat[:, off:off + width].view(flat.shape[0], *shape))
            off += width
        return layers, flat

    def _model_major(self, data):
        layers, flat = self._traces(data)
        return flat[None], [tuple(a.shape[1:]) for a in layers]

    @staticmethod
    def _cam(scores, bits):
        return [np.array(list(P.cam_from_bits(scores[0], bits[0])), dtype=np.int64)]

    def evaluate_all(self, test_dataset, test_dataset_id=None
                     ) -> Tuple[Dict[str, List[float]], Dict[str, np.ndarray], Dict[str, np.ndarray]]:
        """(times, all_scores, cam_orders), each keyed by metric name (handler_coverage.py:103-132).

        times[m] = [setup, pred, quant, cam] in seconds: setup = the metric's debit of the training walk plus its
        construction; pred = collecting and flattening the test set's traces (once, shared by every metric, as the
        reference adds up its per-badge walk for each metric); quant = `metric.packed(...)` with the scores' download;
        cam = `cam_from_bits` on the packed profile.  all_scores[m]: NumPy, in the dtype the reference's `sum_score`
        picks; cam_orders[m]: int64.  Rows are in input order.  test_dataset_id is accepted for the reference's
        signature; nothing is written anywhere.  An empty test set raises ValueError before any launch."""
        return self._evaluate(test_dataset)[0]


def stack_layer_ids(nc_layers: Sequence) -> List[int]:
    """A stack's coverage layers as child indices; ValueError for anything else (a dotted submodule name of a stack
    has no known layout)."""
    ids = list(nc_layers)
    bad = [lid for lid in ids if isinstance(lid, bool) or not isinstance(lid, (int, np.integer))]
    if bad:
        raise ValueError(f"a stack's coverage layers must be child indices, got {bad!r}")
    return [int(lid) for lid in ids]


class StackedCoverageWorker(_CoverageArm):
    """`CoverageWorker` for the M models of a `case_studies.stacked.StackedSequential`, all on the same inputs.

    nc_layers: child indices of the stack (dotted submodule names raise ValueError before any forward pass).
    Training walk: one stacked forward per badge of `batch_size` inputs; every hooked output, turned model-major by
    `stack.model_major`, is fed to one `AggregateStatisticsCollector` as rows [b, M, *layer shape], so one
    `tip_stats_update` per layer and badge serves all M models.  Each neuron's Welford chain is still its own samples
    in order, so model m's statistics (slice m of the collector's, in `self.mins[m]`, `self.maxs[m]`, `self.stds[m]`)
    are bit for bit what the collector gives on model m's traces alone.  NBC, SNAC and KMNC get one object per model
    (`self.metrics[name][m]`), built from that model's statistics; NAC and TKNC hold no state, so one object of each
    serves all M models.

    `evaluate_all(test_dataset)` returns M `(times, scores, orders)` triples in `CoverageWorker.evaluate_all`'s form.
    The test traces go badge by badge into one model-major [M, N, D] buffer; NAC runs once on its [M * N, D] view,
    NBC, SNAC and KMNC on each model's [N, D] slice, TKNC on each model's layer views, and every metric's M profiles
    are ordered by one `prioritizers.cam_from_bits_stack`.  Each phase is timed once for the stack and split evenly
    over the M models (the setup debits are `CoverageWorker`'s, over the stacked walk).

    The scores and orders are those of the single-model metrics on the stack's own traces.  A stacked forward equals
    each model's own forward only to rounding, so they can differ from a `CoverageWorker` on the unstacked model.

    Memory: the buffer takes M * N * D * 4 bytes.  Per model and 10 000 test inputs that is 1.46 GB for the MNIST and
    Fashion-MNIST networks (D = 36 384) and 1.96 GB for CIFAR-10's (D = 49 120); the caller bounds M."""

    def __init__(self, stack, nc_layers: Sequence, training_data, batch_size: int = 128):
        from ..case_studies.stacked import StackedSequential

        if not isinstance(stack, StackedSequential):
            raise ValueError(f"StackedCoverageWorker takes a StackedSequential, got {type(stack).__name__}")
        self.nc_layers = stack_layer_ids(nc_layers)
        self.stack = stack
        self.models = len(stack.sources)
        self.base_model = TransparentModel(stack, self.nc_layers, include_last_layer=False)
        self.batch_size = batch_size
        self.mins, self.maxs, self.stds = self._walk(training_data)
        self.metrics: Dict[str, List[CoverageMethod]] = self._metrics

    def _activations(self, badge):
        """The hooked layers of one stacked forward on `badge` (every model sees it), each [M, b, *layer shape]."""
        acts = self.base_model.get_activations(self.stack.stack_inputs([badge] * self.models))
        return [self.stack.model_major(child, a) for child, a in zip(self.nc_layers, acts)]

    @staticmethod
    def _cam(scores, bits):
        return P.cam_from_bits_stack(list(scores), bits)

    def evaluate_all(self, test_dataset, test_dataset_id=None
                     ) -> List[Tuple[Dict[str, List[float]], Dict[str, np.ndarray], Dict[str, np.ndarray]]]:
        """M (times, all_scores, cam_orders) triples, model m's in `CoverageWorker.evaluate_all`'s form; times[metric]
        = [setup, pred, quant, cam] with each phase's stack time split evenly over the M models.  An empty test set
        raises ValueError before any launch."""
        return self._evaluate(test_dataset)
