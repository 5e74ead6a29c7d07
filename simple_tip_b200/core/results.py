"""On-disk result formats of the reference's prioritization experiments (SURVEY.md §8 f4).

The reference stores every TIP's scores, CAM orders, the misclassification mask and the timings as
flat files whose NAMES carry the meaning (src/dnn_test_prio/eval_prioritization.py:22-58):

    <out>/priorities/<case_study>_<dataset>_<model_id>_<data_type>.npy       np.save / np.load
    <out>/times/<case_study>_<dataset>_<model_id>_<metric>                   pickle of [setup, pred, quant(, cam)]

with data_type in {"is_misclassified", "uncertainty_<quantifier>", "<metric>_scores", "<metric>_cam_order"} and
metric either a surprise adequacy ("dsa", "pc-lsa", ...) or "<CRITERION>_<param>" ("NAC_0.75", "KMNC_2", ...).
`load_apfd_values` re-reads such a folder the way src/plotters/eval_apfd_table.py:43-108 does (scores ->
`np.argsort(-scores)`, CAM orders as stored, APFD against the misclassification mask) — so results written by
this package are consumable by the reference's table scripts and vice versa.  The active-learning experiment's
accuracies go to `<out>/active_learning/<case_study>_<model_id>_<metric>_<nominal|ood>.pickle`
(eval_active_learning.py:134-147, `persist_active_learning`).  Host-side I/O only.
"""
from __future__ import annotations

import os
import pickle
from typing import Dict, List, Optional, Tuple

import numpy as np

from .apfd import apfd_from_order

FIRST_K_MODELS_CONSIDERED = 100            # eval_apfd_table.py:24


def _priorities(output_folder: str) -> str:
    return os.path.join(output_folder, "priorities")


def persist(output_folder: str, case_study: str, dataset_id: str, data_type: str, model_id: int, data) -> str:
    """eval_prioritization.py:22-29 (`_persist`)."""
    os.makedirs(_priorities(output_folder), exist_ok=True)
    path = os.path.join(_priorities(output_folder), f"{case_study}_{dataset_id}_{model_id}_{data_type}.npy")
    np.save(path, np.asarray(data))
    return path


def load(output_folder: str, case_study: str, dataset_id: str, data_type: str, model_id: int) -> np.ndarray:
    """eval_prioritization.py:54-58 (`load`)."""
    return np.load(os.path.join(_priorities(output_folder), f"{case_study}_{dataset_id}_{model_id}_{data_type}.npy"))


def persist_times(output_folder: str, case_study: str, dataset_id: str, model_id: int, metric: str, data: List[float]) -> str:
    """eval_prioritization.py:32-51 (`_persist_times`, `_persist_times_multiple_metrics`: one pickle per metric)."""
    folder = os.path.join(output_folder, "times")
    os.makedirs(folder, exist_ok=True)
    path = os.path.join(folder, f"{case_study}_{dataset_id}_{model_id}_{metric}")
    with open(path, "wb") as f:
        pickle.dump(list(data), f)
    return path


def load_times(output_folder: str, case_study: str, dataset_id: str, model_id: int, metric: str) -> List[float]:
    with open(os.path.join(output_folder, "times", f"{case_study}_{dataset_id}_{model_id}_{metric}"), "rb") as f:
        return pickle.load(f)


def persist_tip(output_folder: str, case_study: str, dataset_id: str, model_id: int, metric: str, scores,
                cam_order=None, times: Optional[List[float]] = None) -> None:
    """Everything one TIP leaves behind for one dataset (eval_prioritization.py:133-154 / :174-193)."""
    persist(output_folder, case_study, dataset_id, f"{metric}_scores", model_id, scores)
    if cam_order is not None:
        persist(output_folder, case_study, dataset_id, f"{metric}_cam_order", model_id, np.array(cam_order))
    if times is not None:
        persist_times(output_folder, case_study, dataset_id, model_id, metric, times)


def persist_active_learning(output_folder: str, case_study: str, model_id: int, metric: str, ood_or_nom: str,
                            eval_res: Dict[Tuple[str, str], float]) -> str:
    """eval_active_learning.py:134-147 (`_save_results_on_file`): one pickle of {(ood_or_nom, observed_or_future):
    accuracy} per retrained model (metric "original", ood_or_nom "na" for the model before retraining), named as
    eval_active_learning_table.py:26-59 expects."""
    folder = os.path.join(output_folder, "active_learning")
    os.makedirs(folder, exist_ok=True)
    path = os.path.join(folder, f"{case_study}_{model_id}_{metric}_{ood_or_nom}.pickle")
    with open(path, "wb") as f:
        pickle.dump(eval_res, f)
    return path


def approach_name(approach: str, param: str = "", cam: bool = False) -> str:
    """src/plotters/utils.py:124-131."""
    return approach + (f"_{param}" if param else "") + ("-cam" if cam else "")


def load_orders(output_folder: str, case_study: str, ds_name: str) -> Tuple[Dict[Tuple[str, str], np.ndarray], Dict[str, np.ndarray]]:
    """(orders[(approach, model_id)], misclassifications[model_id]) parsed from the file names exactly as
    eval_apfd_table.py:56-89 does."""
    misclassifications: Dict[str, np.ndarray] = {}
    orders: Dict[Tuple[str, str], np.ndarray] = {}
    for root, _, files in os.walk(_priorities(output_folder)):
        for file in files:
            if not file.endswith(".npy") or not file.startswith(f"{case_study}_{ds_name}"):
                continue
            arr = np.load(os.path.join(root, file))
            if file.endswith("is_misclassified.npy"):
                _, _, model_id, _, _ = file.split("_")
                if int(model_id) < FIRST_K_MODELS_CONSIDERED:
                    misclassifications[model_id] = arr
            elif file.endswith("cam_order.npy"):
                if "dsa" in file or "lsa" in file:
                    _, _, model_id, metric, _, _ = file.split("_")
                    metric = approach_name(metric, cam=True)
                else:
                    _, _, model_id, metric, param, _, _ = file.split("_")
                    metric = approach_name(metric, param=param, cam=True)
                orders[(metric, model_id)] = arr
            else:
                if "uncertainty" in file:
                    stem = file.replace(".npy", "").replace(f"{case_study}_{ds_name}_", "")
                    model_id, metric = stem.split("_uncertainty_")
                elif "dsa" in file or "lsa" in file:
                    _, _, model_id, metric, _ = file.split("_")
                else:
                    _, _, model_id, metric, param, _ = file.split("_")
                    metric = approach_name(metric, param=param, cam=False)
                orders[(metric, model_id)] = np.argsort(-arr)
    return orders, misclassifications


def load_apfd_values(output_folder: str, case_study: str, ds_name: str) -> Dict[str, Dict[int, float]]:
    """APFD per approach and model id (eval_apfd_table.py:43-108; every approach found on disk is reported)."""
    orders, mis = load_orders(output_folder, case_study, ds_name)
    apfds: Dict[str, Dict[int, float]] = {}
    for (approach, model_id), order in orders.items():
        if model_id not in mis:
            continue
        apfds.setdefault(approach, {})[int(model_id)] = apfd_from_order(mis[model_id], order)
    return apfds
