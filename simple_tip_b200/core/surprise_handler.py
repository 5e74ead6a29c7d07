"""The study's surprise-adequacy arm for PyTorch models (handler_surprise.py:19-117, `SurpriseHandler`).

Collects the training traces and predictions once, fits the five `TESTED_SA` configurations, scores every test set
and orders it by surprise coverage (SC-CAM, `prioritizers.cam_from_surprise`), timing each phase as the reference
does.  The traces come from forward hooks (`activations.TransparentModel`) and stay on the model's device; the
scorers take them from there.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .activations import HookedModelHandler, TransparentModel
from .prioritizers import cam_from_surprise
from .surprise import DSA, LSA, MDSA, MLSA, MultiModalSA, SurpriseCoverageMapper
from .timer import Timer

NUM_SC_BUCKETS = 1000          # handler_surprise.py:14


class SurpriseHandler(HookedModelHandler):
    """`SurpriseHandler(model, sa_layers, training_data)` + `evaluate_all(datasets)` of handler_surprise.py for a
    `torch.nn.Module` whose last output is its softmax.

    sa_layers: as `TransparentModel`'s activation_layers.  Every input set (a tensor or an array [N, ...]) runs
    through the model in batches of `batch_size` on the model's device.  The SAs receive the hooked layers as a list
    of tensors, as the reference passes `outputs[:-1]`: CUDA tensors stay on the device, host tensors become NumPy
    arrays.  The predictions are the first-index argmax of the last output (`np.argmax`'s tie rule), computed by
    torch on the model's device and handed over as host int64.

    The SAs' fit backends follow the B200TIP_KDE / B200TIP_COV / B200TIP_GMM / B200TIP_KMEANS variables.  Scores are
    NumPy arrays in the SA's dtype.  Every timer ends with a synchronise of the current CUDA device (and the model's,
    when that is another one), so device work is inside the phase that launched it.

    Writing the reference's result files (eval_prioritization.py:114-154; `prioritization.evaluate` runs the whole
    experiment, this arm included):

        res = SurpriseHandler(model, [3], x_train).evaluate_all({"nominal": x_test, "ood": x_ood})
        for sa_name, per_ds in res.items():
            for ds_name, (scores, cam_order, times) in per_ds.items():
                results.persist_tip(out, case_study, ds_name, model_id, sa_name, scores, cam_order, times)
    """

    TESTED_SA = {
        # handler_surprise.py:22-37
        "dsa": lambda x, y: DSA(x, y, subsampling=0.3),
        "pc-lsa": lambda x, y: MultiModalSA.build_by_class(x, y, lambda x, y: LSA(x)),
        "pc-mdsa": lambda x, y: MultiModalSA.build_by_class(x, y, lambda x, y: MDSA(x)),
        "pc-mlsa": lambda x, y: MultiModalSA.build_by_class(x, y, lambda x, y: MLSA(x, num_components=3)),
        "pc-mmdsa": lambda x, y: MultiModalSA.build_with_kmeans(x, y, lambda x, y: MDSA(x), potential_k=range(2, 6),
                                                                subsampling=0.3),
    }

    def __init__(self, model, sa_layers: Sequence, training_data, batch_size: int = 128):
        self.sa_layers = list(sa_layers)
        self.base_model = TransparentModel(model, self.sa_layers, include_last_layer=True)
        self.batch_size = batch_size
        self.train_at_timer = Timer()
        self.train_ats, self.train_pred = self._synced(lambda: self._acti_and_pred(training_data),
                                                       self.train_at_timer)

    def _acti_and_pred(self, data) -> Tuple[List, np.ndarray]:
        """handler_surprise.py:51-57: the hooked layers and the predictions of one forward pass."""
        import torch

        x = data if isinstance(data, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(data))
        outputs = self.base_model.collect(x.to(self._model_device()), self.batch_size)
        assert len(outputs) == len(self.sa_layers) + 1
        ats = [a if a.is_cuda else a.numpy() for a in outputs[:-1]]
        return ats, outputs[-1].argmax(dim=1).cpu().numpy().astype(np.int64)

    def evaluate_all(self, datasets: Dict[str, object], dsa_badge_size: Optional[int] = None
                     ) -> Dict[str, Dict[str, Tuple[np.ndarray, np.ndarray, List[float]]]]:
        """{sa_name: {ds_name: (scores, cam_order, [setup, pred, sa, cam])}} (handler_surprise.py:59-117): setup =
        the training traces' time plus the SA's fit, pred = the test set's traces, sa = scoring, cam = SC-CAM with
        NUM_SC_BUCKETS buckets up to the largest score.  `dsa_badge_size` sets DSA's `badge_size`."""
        res: Dict[str, Dict[str, Tuple]] = {}
        test_apt = {}
        for ds_name, data in datasets.items():
            timer = Timer()
            ats, pred = self._synced(lambda: self._acti_and_pred(data), timer)
            test_apt[ds_name] = (ats, pred, timer.get())

        for sa_name, sa_func in self.TESTED_SA.items():
            res[sa_name] = {}

            def setup():
                sa = sa_func(self.train_ats, self.train_pred)
                if isinstance(sa, DSA) and dsa_badge_size is not None:
                    sa.badge_size = dsa_badge_size
                return sa
            setup_timer = Timer()
            sa = self._synced(setup, setup_timer)
            setup_time = self.train_at_timer.get() + setup_timer.get()
            for ds_name, (ats, pred, pred_time) in test_apt.items():
                sa_timer = Timer()
                scores = self._synced(lambda: sa(ats, pred), sa_timer)
                res[sa_name][ds_name] = (scores, [setup_time, pred_time, sa_timer.get()])

        for sa_name in self.TESTED_SA:
            for ds_name in datasets:
                scores, times = res[sa_name][ds_name]
                cam_timer = Timer()
                order = self._synced(lambda: np.array(list(cam_from_surprise(
                    scores, SurpriseCoverageMapper(NUM_SC_BUCKETS, np.max(scores))))), cam_timer)
                times.append(cam_timer.get())
                res[sa_name][ds_name] = (scores, order, times)
        return res
