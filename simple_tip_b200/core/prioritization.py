"""The study's test-prioritization experiment for PyTorch models (eval_prioritization.py:62-215, `evaluate`).

Runs the three arms on the nominal and the out-of-distribution test set in the reference's order — the fault
predictors (`activations.get_pred_and_uncertainty`), the neuron-coverage arm (`coverage_worker.CoverageWorker`) and
the surprise arm (`surprise_handler.SurpriseHandler`) — and writes every score, CAM order, misclassification mask
and time file the reference writes (`results.persist`, `persist_times`, `persist_tip`), so the reference's
`src/plotters/eval_apfd_table.py` and `results.apfd_table` read them unchanged.

CUDA tensors stay on their device; the arms move host inputs to the model's device.  The APFDs are host NumPy, as in
the reference's table script: the arms return host scores, and for tied scores `np.argsort`'s tie order decides the
APFD.
"""
from __future__ import annotations

import gc
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import activations, coverage_worker, results, surprise_handler

NOM = "nominal"
OOD = "ood"

OUTPUT_FOLDER = "/assets/"        # case_study.py:10

Arrays = Dict[str, np.ndarray]
"""{approach: scores or CAM order} of one dataset"""


def evaluate(model_id: int, case_study: str, model, training_dataset, nominal_test_dataset, nominal_test_labels,
             ood_test_dataset, ood_test_labels, nc_activation_layers: Sequence, sa_activation_layers: Sequence,
             dsa_badge_size: Optional[int] = None, output_folder: str = OUTPUT_FOLDER, batch_size: int = 128
             ) -> Dict[str, Dict[str, float]]:
    """eval_prioritization.py:62-111 for a `torch.nn.Module` whose last output is its softmax.

    The datasets are NumPy arrays or torch tensors [N, ...] (host or CUDA); the labels hold one entry per input, as
    [N] or [N, 1], and are flattened.  The layers are as `TransparentModel`'s activation_layers; `batch_size` is the
    badge size of the coverage and the surprise arm (the fault predictors run with `get_pred_and_uncertainty`'s
    defaults).  The result files go to `{output_folder}/priorities/` and `{output_folder}/times/` (created when
    missing).  The model is left as it was: its parameters untouched, every module's training flag restored.

    Returns {"nominal" / "ood": {approach: APFD}} for the approaches of the study's table (`results.APPROACHES`)
    that were scored: all 39, or 38 when the model has no dropout module (no VR).  Each value is the one
    `results.load_apfd_values(output_folder, case_study, ds)[approach][model_id]` reads back; the reference returns
    None.  ValueError before any forward pass when a label array does not hold one entry per input, or when
    `case_study` contains "_" (the table script splits the file names at "_")."""
    if "_" in case_study:
        raise ValueError(f"case_study {case_study!r} contains '_', which the result file names cannot carry")
    labels = {NOM: _flat_labels(nominal_test_labels, nominal_test_dataset, "nominal_test_labels"),
              OOD: _flat_labels(ood_test_labels, ood_test_dataset, "ood_test_labels")}
    datasets = {NOM: nominal_test_dataset, OOD: ood_test_dataset}

    masks: Dict[str, np.ndarray] = {}
    scores: Dict[str, Arrays] = {NOM: {}, OOD: {}}
    cam_orders: Dict[str, Arrays] = {NOM: {}, OOD: {}}
    for ds in (NOM, OOD):
        masks[ds], scores[ds] = _eval_fault_predictors(output_folder, case_study, model, model_id, datasets[ds],
                                                       labels[ds], ds)

    # each arm's worker lives in its helper only, so the coverage traces are freed before the surprise handler's
    nc_scores, nc_orders = _eval_neuron_coverage(output_folder, case_study, model, model_id, datasets,
                                                 training_dataset, nc_activation_layers, batch_size)
    gc.collect()
    sa_scores, sa_orders = _eval_surprise(output_folder, case_study, model, model_id, datasets, training_dataset,
                                          sa_activation_layers, batch_size, dsa_badge_size)
    gc.collect()
    for ds in (NOM, OOD):
        scores[ds].update(nc_scores[ds])
        scores[ds].update(sa_scores[ds])
        cam_orders[ds].update(nc_orders[ds])
        cam_orders[ds].update(sa_orders[ds])

    res: Dict[str, Dict[str, float]] = {}
    for ds in (NOM, OOD):
        apfds = results.apfd_values(masks[ds], scores[ds], cam_orders[ds])
        res[ds] = {approach: apfds[approach] for approach in results.APPROACHES if approach in apfds}
    return res


def evaluate_stack(model_ids: Sequence[int], case_study: str, models: Sequence, training_dataset,
                   nominal_test_dataset, nominal_test_labels, ood_test_dataset, ood_test_labels,
                   nc_activation_layers: Sequence, sa_activation_layers: Sequence,
                   dsa_badge_size: Optional[int] = None, output_folder: str = OUTPUT_FOLDER, batch_size: int = 128,
                   stacked_coverage: bool = False) -> Dict[int, Dict[str, Dict[str, float]]]:
    """`evaluate` for M models of one architecture (`KerasSequential` networks, model k has id model_ids[k]):
    every file `evaluate(model_ids[k], ..., models[k], ...)` writes, under the same names.

    The fault predictors of both datasets come from one `case_studies.stacked.stack(models)`
    (`activations.get_pred_and_uncertainty_stack`, its defaults as `evaluate` takes the single-model ones); by default
    the coverage and the surprise arm then run model by model, in `evaluate`'s order, each arm freed before the next.
    Their score and CAM-order files are those of `evaluate`; the fault predictors' are those of the stacked forward,
    which equals each model's own forward to rounding (the torch sampler's masks differ: see
    `get_pred_and_uncertainty_stack`), and their time files hold each phase's time split evenly over the M models.

    stacked_coverage=True runs the coverage arm on the stack too: one `coverage_worker.StackedCoverageWorker` walks
    the training set once for all M models and scores both datasets, writing every coverage file `evaluate` writes
    under the same names.  Its traces are the stacked forward's, so its scores and orders equal `evaluate`'s only as
    far as that forward's rounding allows, and its time files hold each phase's time split evenly over the M models.
    The surprise arm still runs model by model.

    Returns {model_id: what `evaluate` returns for it}.  ValueError, before any forward pass, for the conditions
    `evaluate` refuses, for len(models) != len(model_ids), for repeated model ids and, with stacked_coverage, for
    coverage layers that are not child indices."""
    from ..case_studies.stacked import stack

    model_ids = [int(i) for i in model_ids]
    if len(model_ids) != len(models):
        raise ValueError(f"{len(model_ids)} model ids for {len(models)} models")
    if len(set(model_ids)) != len(model_ids):
        raise ValueError(f"model ids {model_ids} repeat")
    if "_" in case_study:
        raise ValueError(f"case_study {case_study!r} contains '_', which the result file names cannot carry")
    if stacked_coverage:
        coverage_worker.stack_layer_ids(nc_activation_layers)
    labels = {NOM: _flat_labels(nominal_test_labels, nominal_test_dataset, "nominal_test_labels"),
              OOD: _flat_labels(ood_test_labels, ood_test_dataset, "ood_test_labels")}
    datasets = {NOM: nominal_test_dataset, OOD: ood_test_dataset}

    masks: Dict[int, Dict[str, np.ndarray]] = {i: {} for i in model_ids}
    scores: Dict[int, Dict[str, Arrays]] = {i: {NOM: {}, OOD: {}} for i in model_ids}
    cam_orders: Dict[int, Dict[str, Arrays]] = {i: {NOM: {}, OOD: {}} for i in model_ids}
    stacked = stack(models)
    for ds in (NOM, OOD):
        per_model = activations.get_pred_and_uncertainty_stack(stacked, datasets[ds])
        for model_id, (pred, uncertainties, times) in zip(model_ids, per_model):
            masks[model_id][ds], scores[model_id][ds] = _persist_fault_predictors(
                output_folder, case_study, model_id, labels[ds], ds, pred, uncertainties, times)
    del per_model
    stacked_nc = (_eval_neuron_coverage_stack(output_folder, case_study, stacked, model_ids, datasets, training_dataset,
                                              nc_activation_layers, batch_size) if stacked_coverage else None)
    del stacked
    gc.collect()

    res: Dict[int, Dict[str, Dict[str, float]]] = {}
    for k, (model_id, model) in enumerate(zip(model_ids, models)):
        if stacked_nc is not None:
            nc_scores, nc_orders = stacked_nc[k]
        else:
            nc_scores, nc_orders = _eval_neuron_coverage(output_folder, case_study, model, model_id, datasets,
                                                         training_dataset, nc_activation_layers, batch_size)
            gc.collect()
        sa_scores, sa_orders = _eval_surprise(output_folder, case_study, model, model_id, datasets, training_dataset,
                                              sa_activation_layers, batch_size, dsa_badge_size)
        gc.collect()
        res[model_id] = {}
        for ds in (NOM, OOD):
            scores[model_id][ds].update(nc_scores[ds])
            scores[model_id][ds].update(sa_scores[ds])
            cam_orders[model_id][ds].update(nc_orders[ds])
            cam_orders[model_id][ds].update(sa_orders[ds])
            apfds = results.apfd_values(masks[model_id][ds], scores[model_id][ds], cam_orders[model_id][ds])
            res[model_id][ds] = {approach: apfds[approach] for approach in results.APPROACHES if approach in apfds}
    return res


def _host(a) -> np.ndarray:
    try:
        import torch
    except ImportError:      # pragma: no cover
        torch = None
    if torch is not None and isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _flat_labels(labels, data, what: str) -> np.ndarray:
    """labels [N] or [N, 1] of the N inputs of `data` as a flat host array; ValueError otherwise (the reference's
    `pred != labels` would broadcast [N, 1] against [N] to an [N, N] mask)."""
    y = _host(labels)
    n = int(data.shape[0])
    if y.ndim == 0 or y.shape[0] != n or y.size != n:
        raise ValueError(f"{what} holds {tuple(y.shape)} labels for {n} inputs; expected [{n}] or [{n}, 1]")
    return y.reshape(-1)


def _eval_fault_predictors(output_folder, case_study, model, model_id, x, labels, ds) -> Tuple[np.ndarray, Arrays]:
    """eval_prioritization.py:193-215: the misclassification mask, every quantifier's uncertainties and times."""
    pred, uncertainties, times = activations.get_pred_and_uncertainty(model, x)
    return _persist_fault_predictors(output_folder, case_study, model_id, labels, ds, pred, uncertainties, times)


def _persist_fault_predictors(output_folder, case_study, model_id, labels, ds, pred, uncertainties, times
                              ) -> Tuple[np.ndarray, Arrays]:
    is_misclassified = pred != labels
    results.persist(output_folder, case_study, ds, "is_misclassified", model_id, is_misclassified)
    for metric, t in times.items():
        results.persist_times(output_folder, case_study, ds, model_id, metric, t)
    for metric, unc in uncertainties.items():
        results.persist(output_folder, case_study, ds, f"uncertainty_{metric}", model_id, unc)
    return is_misclassified, dict(uncertainties)


def _eval_neuron_coverage(output_folder, case_study, model, model_id, datasets, training_dataset, layers,
                          batch_size) -> Tuple[Dict[str, Arrays], Dict[str, Arrays]]:
    """eval_prioritization.py:157-190: the twelve coverage metrics' scores, CAM orders and times per dataset."""
    scores: Dict[str, Arrays] = {}
    cam_orders: Dict[str, Arrays] = {}
    nc_worker = coverage_worker.CoverageWorker(model, layers, training_dataset, batch_size=batch_size)
    for ds, x in datasets.items():
        times, all_scores, orders = nc_worker.evaluate_all(x, ds)
        for metric, s in all_scores.items():
            results.persist_tip(output_folder, case_study, ds, model_id, metric, s, orders[metric], times[metric])
        scores[ds] = dict(all_scores)
        cam_orders[ds] = {f"{metric}-cam": np.array(order) for metric, order in orders.items()}
    return scores, cam_orders


def _eval_neuron_coverage_stack(output_folder, case_study, stacked, model_ids, datasets, training_dataset, layers,
                                batch_size) -> List[Tuple[Dict[str, Arrays], Dict[str, Arrays]]]:
    """`_eval_neuron_coverage` for every model of a stack from one `StackedCoverageWorker`: per model (in stack
    order) its scores and CAM orders per dataset, its files written under its id."""
    per_model = [({}, {}) for _ in model_ids]
    nc_worker = coverage_worker.StackedCoverageWorker(stacked, layers, training_dataset, batch_size=batch_size)
    for ds, x in datasets.items():
        for (scores, cam_orders), model_id, (times, all_scores, orders) in zip(per_model, model_ids,
                                                                             nc_worker.evaluate_all(x, ds)):
            for metric, s in all_scores.items():
                results.persist_tip(output_folder, case_study, ds, model_id, metric, s, orders[metric], times[metric])
            scores[ds] = dict(all_scores)
            cam_orders[ds] = {f"{metric}-cam": np.array(order) for metric, order in orders.items()}
    return per_model


def _eval_surprise(output_folder, case_study, model, model_id, datasets, training_dataset, layers, batch_size,
                   dsa_badge_size) -> Tuple[Dict[str, Arrays], Dict[str, Arrays]]:
    """eval_prioritization.py:114-154: the five surprise adequacies' scores, SC-CAM orders and times per dataset."""
    scores: Dict[str, Arrays] = {ds: {} for ds in datasets}
    cam_orders: Dict[str, Arrays] = {ds: {} for ds in datasets}
    sa_worker = surprise_handler.SurpriseHandler(model, layers, training_dataset, batch_size=batch_size)
    sa_results = sa_worker.evaluate_all(dict(datasets), dsa_badge_size=dsa_badge_size)
    for metric, values in sa_results.items():
        for ds, (sa, cam_order, times) in values.items():
            results.persist_tip(output_folder, case_study, ds, model_id, metric, sa, cam_order, times)
            scores[ds][metric] = sa
            cam_orders[ds][f"{metric}-cam"] = np.array(cam_order)
    return scores, cam_orders
