"""The study's active-learning experiment for PyTorch models (eval_active_learning.py:34-313, `evaluate`).

Splits the nominal and the out-of-distribution test sets into an observed and a future half, asks every TIP of the
three arms for its selection on the observed halves (`activations.get_pred_and_uncertainty`,
`coverage_worker.CoverageWorker`, `surprise_handler.SurpriseHandler`) plus the random baseline, retrains once per
selection through the caller's `training_process`, and scores the original and every retrained model on all four
splits.  The accuracies go to disk as the reference writes them (`results.persist_active_learning`), so the
reference's `src/plotters/eval_active_learning_table.py` reads them unchanged.

CUDA tensors stay on their device the whole way: the splits, the selected rows and the retraining set are gathered
and concatenated there.  The selections themselves are host NumPy, as in the reference: the arms return host scores,
and `np.argsort`'s tie order is what decides which of equally scored inputs is selected.
"""
from __future__ import annotations

import gc
from typing import Callable, Dict, Optional, Sequence, Tuple

import numpy as np

from . import activations, coverage_worker, results, surprise_handler

RANDOM_SPLIT = "random"

SplitDataset = Dict[Tuple[str, str], Tuple[object, object]]
"""{("nominal" / "ood", "observed" / "future"): (x, y)}"""

SplitEvaluation = Dict[Tuple[str, str], float]
"""{("nominal" / "ood", "observed" / "future"): accuracy}"""

MetricSelection = Dict[Tuple[str, str], object]
"""{(metric, "nominal" / "ood"): selected indexes into the observed split}"""

NOM = "nominal"
OOD = "ood"

OBS = "observed"
FUT = "future"

OUTPUT_FOLDER = "/assets/"        # case_study.py:10


def evaluate(model_id: int, case_study: str, model, train_x, train_y, nominal_test_x, nominal_test_labels,
             ood_test_x, ood_test_labels, nc_activation_layers: Sequence, sa_activation_layers: Sequence,
             training_process: Optional[Callable], observed_share: float, num_selected: int,
             num_classes: Optional[int], dsa_badge_size: Optional[int] = None, output_folder: str = OUTPUT_FOLDER,
             batch_size: int = 128, stacked_training_process: Optional[Callable] = None
             ) -> Tuple[SplitEvaluation, MetricSelection, Dict[Tuple[str, str], SplitEvaluation]]:
    """eval_active_learning.py:34-131 for a `torch.nn.Module` whose last output is its softmax.

    Inputs are NumPy arrays or torch tensors (host or CUDA).  `training_process(x, y)` receives torch tensors — on
    the inputs' device when they are CUDA tensors — with `y` float32 one-hot when `num_classes` is given, else the
    flattened labels; it returns a `torch.nn.Module`.  The layers are as `TransparentModel`'s activation_layers;
    `batch_size` is the badge size of the arms' forward passes and of the accuracy evaluation.  The result files go
    to `{output_folder}/active_learning/` (created when missing).

    `stacked_training_process(x_pool, y_pool, rows)`, when given, retrains every selection's model in one call
    instead (and `training_process` may be None): x_pool is the training set followed by the nominal and the OOD
    observed split, concatenated once on the inputs' device (a torch tensor), y_pool their labels the same way (one-hot
    as above, on x_pool's device), and rows the int64 [selections, n] tensor of pool rows on that device whose row k
    is exactly the retraining set `training_process` would receive for selection k (`np.random.permutation` is drawn
    once per selection, in the same order).  It returns the retrained models in selection order.  When they are
    `KerasSequential` networks of one architecture (a case study's `stacked_training_process`), they are evaluated
    together, one stacked forward per badge and split (`accuracies_stack`); other modules are evaluated one by one
    as the sequential loop evaluates them.

    Returns (original model's accuracies, selections, {(metric, "nominal" / "ood"): retrained model's accuracies}),
    each dict in the reference's insertion order; the reference returns None."""
    active_datasets = _shuffle_and_split_datasets(model_id, nominal_test_x, nominal_test_labels, ood_test_x,
                                                  ood_test_labels, observed_share=observed_share)

    original_model_eval = _evaluate(model, active_datasets, num_classes, batch_size)

    # each arm's worker lives in its helper only, so its traces are freed before the first retraining
    selections: MetricSelection = dict()
    selections.update(_get_fp_selection(model, active_datasets, num_selected))
    selections.update(_get_nc_selection(model, train_x, active_datasets, nc_activation_layers, num_selected,
                                        batch_size))
    selections.update(_get_sa_selection(model, train_x, active_datasets, sa_activation_layers, num_selected,
                                        dsa_badge_size, batch_size))
    selections.update(_get_random_section(active_datasets, num_selected))
    gc.collect()

    _selection_sanity_checks(num_selected, selections)

    active_accuracies: Dict[Tuple[str, str], SplitEvaluation] = dict()
    if stacked_training_process is not None:
        new_models = _retrain_stacked(num_classes, stacked_training_process, train_x, train_y, active_datasets,
                                      selections)
        for key, eval_res in zip(selections, _evaluate_stack(new_models, active_datasets, num_classes, batch_size)):
            active_accuracies[key] = eval_res
        del new_models
    else:
        for (metric, ood_or_nom), selected_indexes in selections.items():
            x, y = active_datasets[ood_or_nom, OBS]
            new_model = _retrain(num_classes, training_process, train_x, train_y, _take(x, selected_indexes),
                                 _take(y, selected_indexes))
            # every model is evaluated on all four splits, as in the reference (:104-109)
            active_accuracies[(metric, ood_or_nom)] = _evaluate(new_model, active_datasets, num_classes, batch_size)
            del new_model

    results.persist_active_learning(output_folder, case_study, model_id, "original", "na", original_model_eval)
    for (metric, ood_or_nom), eval_res in active_accuracies.items():
        results.persist_active_learning(output_folder, case_study, model_id, metric, ood_or_nom, eval_res)
    return original_model_eval, selections, active_accuracies


def _is_tensor(a) -> bool:
    try:
        import torch
    except ImportError:      # pragma: no cover
        return False
    return isinstance(a, torch.Tensor)


def _take(a, idx):
    """Rows `idx` (any integer sequence) of an array or a tensor, on the device `a` lives on."""
    idx = np.asarray(idx, dtype=np.int64)
    if _is_tensor(a):
        import torch

        return a[torch.from_numpy(idx).to(a.device)]
    return a[idx]


def _as_tensor(a, device=None):
    import torch

    t = a if _is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    return t if device is None else t.to(device)


def _concat(a, b):
    """np.concatenate((a, b)) for two arrays; for a tensor among them, torch.cat on the device of the first CUDA
    operand (else the host)."""
    if not _is_tensor(a) and not _is_tensor(b):
        return np.concatenate((a, b))
    import torch

    devices = [t.device for t in (a, b) if _is_tensor(t) and t.is_cuda]
    device = devices[0] if devices else torch.device("cpu")
    return torch.cat((_as_tensor(a, device), _as_tensor(b, device)))


def _selection_sanity_checks(num_selected, selections):
    """eval_active_learning.py:150-158."""
    for (metric, ood_or_nom), selected_idx in selections.items():
        assert len(selected_idx) == num_selected, (
            f"The number of selected indexes for {metric}, {ood_or_nom} is not correct."
            f"Should be {num_selected}, but was {len(selected_idx)}"
        )
        assert (
            len(set(selected_idx)) == num_selected
        ), f"The number of selected indexes for {metric}, {ood_or_nom} is not unique."


def _one_hot(y, num_classes: int):
    """keras.utils.to_categorical(y, num_classes) of flat integer labels: float32 [n, num_classes], on y's device."""
    import torch

    y = y.to(torch.int64)
    out = torch.zeros((y.shape[0], num_classes), dtype=torch.float32, device=y.device)
    return out.scatter_(1, y.unsqueeze(1), 1.0)


def _retrain(num_classes, training_process, train_x, train_y, new_x, new_y):
    """eval_active_learning.py:161-180: the training set plus the selected rows, shuffled by the global NumPy RNG."""
    x = _concat(train_x, new_x)

    # Make sure we do not flatten away non-empty dimensions,
    #   which would indicate a bug in the code
    assert train_y.shape[0] == np.prod(train_y.shape)
    assert new_y.shape[0] == np.prod(new_y.shape)
    y = _concat(train_y.reshape(-1), new_y.reshape(-1))
    shuffled_idx = np.random.permutation(len(x))
    x, y = _as_tensor(_take(x, shuffled_idx)), _as_tensor(_take(y, shuffled_idx))
    if num_classes is not None:
        y = _one_hot(y, num_classes)
    return training_process(x, y)


def _retrain_stacked(num_classes, stacked_training_process, train_x, train_y, datasets: SplitDataset,
                     selections: MetricSelection) -> list:
    """`_retrain` for every selection in one `stacked_training_process(x_pool, y_pool, rows)` call: the pool is the
    training set followed by the two observed splits, and rows[k] maps selection k's merged set, shuffled by the
    same global-RNG draw `_retrain` takes, to pool rows, so x_pool[rows[k]] is what `_retrain` would hand over."""
    import torch

    assert train_y.shape[0] == np.prod(train_y.shape)
    x_pool, y_pool, offset = train_x, train_y.reshape(-1), {}
    n = len(train_x)
    for name in (NOM, OOD):
        x, y = datasets[name, OBS]
        assert y.shape[0] == np.prod(y.shape)
        offset[name] = n
        n += len(x)
        x_pool, y_pool = _concat(x_pool, x), _concat(y_pool, y.reshape(-1))
    x_pool = _as_tensor(x_pool)
    y_pool = _as_tensor(y_pool, x_pool.device)
    if num_classes is not None:
        y_pool = _one_hot(y_pool, num_classes)
    train_rows = np.arange(len(train_x), dtype=np.int64)
    rows = []
    for (_, ood_or_nom), selected_indexes in selections.items():
        merged = np.concatenate((train_rows, offset[ood_or_nom] + np.asarray(selected_indexes, dtype=np.int64)))
        rows.append(merged[np.random.permutation(len(merged))])
    rows = torch.from_numpy(np.stack(rows)).to(x_pool.device)
    return list(stacked_training_process(x_pool, y_pool, rows))


def _get_random_section(dataset: SplitDataset, num_selected: int) -> MetricSelection:
    """eval_active_learning.py:183-190: the observed splits are already shuffled."""
    res: MetricSelection = dict()
    for (ood_or_nom, observed_or_future), _ in dataset.items():
        if observed_or_future == OBS:
            res[RANDOM_SPLIT, ood_or_nom] = [x for x in range(num_selected)]
    return res


def _get_fp_selection(model, datasets: SplitDataset, num_selected: int) -> MetricSelection:
    """eval_active_learning.py:193-209: the most uncertain inputs per quantifier."""
    res: MetricSelection = dict()
    for (ood_or_nom, observed_or_future), (x, _) in datasets.items():
        if observed_or_future == OBS:
            _, uncertainties, _ = activations.get_pred_and_uncertainty(model, x)
            for metric, uncertainty in uncertainties.items():
                res[metric, ood_or_nom] = np.argsort(uncertainty)[-num_selected:]
    return res


def _get_nc_selection(model, train_x, datasets: SplitDataset, nc_activation_layers: Sequence, num_selected: int,
                      batch_size: int = 128) -> MetricSelection:
    """eval_active_learning.py:212-239: the highest coverage scores, and the head of each CAM order."""
    res: MetricSelection = dict()
    nc_worker = coverage_worker.CoverageWorker(model, nc_activation_layers, train_x, batch_size=batch_size)
    for (ood_or_nom, observed_or_future), (x, _) in datasets.items():
        if observed_or_future == OBS:
            _, all_scores, cam_orders = nc_worker.evaluate_all(x, num_selected)
            for metric, scores in all_scores.items():
                res[metric, ood_or_nom] = np.argsort(scores)[-num_selected:]
            for metric, cam_order in cam_orders.items():
                res[f"{metric}-cam", ood_or_nom] = cam_order[:num_selected]
    return res


def _get_sa_selection(model, train_x, datasets: SplitDataset, sa_activation_layers: Sequence, num_selected: int,
                      dsa_badge_size: Optional[int] = None, batch_size: int = 128) -> MetricSelection:
    """eval_active_learning.py:242-270: the highest surprise adequacies, and the head of each SC-CAM order."""
    res: MetricSelection = dict()
    sa_worker = surprise_handler.SurpriseHandler(model, sa_activation_layers, train_x, batch_size=batch_size)
    sa_results = sa_worker.evaluate_all({NOM: datasets[NOM, OBS][0], OOD: datasets[OOD, OBS][0]},
                                        dsa_badge_size=dsa_badge_size)
    for metric, values in sa_results.items():
        for nom_or_ood, (sa, cam_order, _) in values.items():
            res[metric, nom_or_ood] = np.argsort(sa)[-num_selected:]
            res[f"{metric}-cam", nom_or_ood] = cam_order[:num_selected]
    return res


def split_indices(n: int, observed_share: float, model_id: int) -> Tuple[np.ndarray, np.ndarray]:
    """(observed, future) row indices of a test set of n rows: the test and the train part of sklearn's
    `train_test_split(..., test_size=observed_share, random_state=model_id)`, which depend on n only."""
    from sklearn.model_selection import train_test_split

    fut, obs = train_test_split(np.arange(n), test_size=observed_share, random_state=model_id)
    return obs, fut


def _shuffle_and_split_datasets(model_id: int, nominal_x, nominal_y, ood_x, ood_y, observed_share: float
                                ) -> SplitDataset:
    """eval_active_learning.py:273-296, each split gathered on the device its set lives on."""
    res: SplitDataset = dict()
    for name, x, y in ((NOM, nominal_x, nominal_y), (OOD, ood_x, ood_y)):
        obs, fut = split_indices(len(x), observed_share, model_id)
        res[name, OBS] = (_take(x, obs), _take(y, obs))
        res[name, FUT] = (_take(x, fut), _take(y, fut))
    return res


def accuracy(model, x, y, batch_size: int = 128) -> float:
    """What Keras' `model.evaluate(x, y)[1]` is for the study's softmax models: the share of inputs whose first-index
    argmax of the output equals the label, as the exact `correct / n`.  The model runs where its parameters live,
    in eval mode without gradients, in batches of `batch_size`; its modes are restored afterwards."""
    return _accuracies(model, 1, lambda xb: model(xb)[None], x, y, batch_size)[0]


def accuracies_stack(stack, x, y, batch_size: int = 128) -> list:
    """`accuracy` of each of the M models of a `StackedSequential` (`case_studies.stacked.stack`) on the same (x, y),
    from one stacked forward per batch of `batch_size`: model m's exact correct / n, its correct count summed from the
    first-index argmax of its slice [b, classes] of the stacked softmax output.  The stack runs in eval mode without
    gradients; its modes are restored afterwards."""
    m = len(stack.sources)
    return _accuracies(stack, m, lambda xb: stack(stack.stack_inputs([xb] * m)), x, y, batch_size)


def _accuracies(model, models: int, forward, x, y, batch_size: int) -> list:
    """Each model's exact correct / n, where forward(batch) gives the M = `models` outputs [M, b, classes] of
    `model`, which runs in eval mode without gradients and has its modes restored afterwards."""
    import torch

    dev = next(iter(model.parameters()), torch.empty(0)).device
    labels = _as_tensor(y, dev).reshape(-1)
    n = labels.shape[0]
    modes = [(module, module.training) for module in model.modules()]
    correct = torch.zeros(models, dtype=torch.int64, device=dev)
    model.eval()
    try:
        with torch.no_grad():
            for start in range(0, n, batch_size):
                out = forward(_as_tensor(x[start:start + batch_size], dev))
                correct += (out.argmax(dim=2) == labels[start:start + batch_size]).sum(dim=1)
    finally:
        for module, training in modes:
            module.training = training
    return [int(c) / n for c in correct.tolist()]


def _checked(acc: float) -> float:
    assert 0 <= acc <= 1, (
        "The models metric is not accuracy, change your "
        "training_process callable."
    )
    return acc


def _evaluate_stack(models: Sequence, datasets: SplitDataset, num_classes: Optional[int], batch_size: int = 128
                    ) -> list:
    """`_evaluate` of every model, one SplitEvaluation per model in order.  `KerasSequential` networks of one
    architecture (what a case study's `stacked_training_process` returns) are scored together, one stacked forward
    per batch and split (`accuracies_stack`); any other modules one by one with `_evaluate`."""
    from ..case_studies.base import KerasSequential
    from ..case_studies.stacked import stack

    if not models or not all(isinstance(m, KerasSequential) for m in models):
        return [_evaluate(m, datasets, num_classes, batch_size) for m in models]
    net = stack(models)
    res = [dict() for _ in models]
    for key, (x, y) in datasets.items():
        for eval_res, acc in zip(res, accuracies_stack(net, x, y, batch_size)):
            eval_res[key] = _checked(acc)
    return res


def _evaluate(model, datasets: SplitDataset, num_classes: Optional[int], batch_size: int = 128) -> SplitEvaluation:
    """eval_active_learning.py:299-313: the model's accuracy on all four splits."""
    return {key: _checked(accuracy(model, x, y, batch_size)) for key, (x, y) in datasets.items()}
