"""On-disk result formats of the reference's prioritization experiments (SURVEY.md §8 f4).

The reference stores every TIP's scores, CAM orders, the misclassification mask and the timings as
flat files whose NAMES carry the meaning (src/dnn_test_prio/eval_prioritization.py:22-58):

    <out>/priorities/<case_study>_<dataset>_<model_id>_<data_type>.npy       np.save / np.load
    <out>/times/<case_study>_<dataset>_<model_id>_<metric>                   pickle of [setup, pred, quant(, cam)]

with data_type in {"is_misclassified", "uncertainty_<quantifier>", "<metric>_scores", "<metric>_cam_order"} and
metric either a surprise adequacy ("dsa", "pc-lsa", ...) or "<CRITERION>_<param>" ("NAC_0.75", "KMNC_2", ...).
`load_apfd_values` re-reads such a folder the way src/plotters/eval_apfd_table.py:43-108 does (scores ->
`np.argsort(-scores)`, CAM orders as stored, APFD against the misclassification mask) — so results written by
this package are consumable by the reference's table scripts and vice versa; `apfd_values` is that rating for one
model's arrays, shared with `prioritization.evaluate`.  `apfd_table` / `write_apfd_table` build the study's Table 1
from such a folder as src/plotters/eval_apfd_table.py does, without TensorFlow.  The active-learning experiment's
accuracies go to `<out>/active_learning/<case_study>_<model_id>_<metric>_<nominal|ood>.pickle`
(eval_active_learning.py:134-147, `persist_active_learning`).  Host-side I/O only.
"""
from __future__ import annotations

import os
import pickle
import statistics
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

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


MISCLASSIFIED, SCORES, CAM_ORDER = "is_misclassified", "scores", "cam_order"


def _priority_files(output_folder: str, case_study: str, ds_name: str) -> Iterator[Tuple[str, str, str, np.ndarray]]:
    """(kind, approach, model_id, array) of every priority file of one case study and dataset, in `os.walk`'s order,
    parsed from the file names exactly as eval_apfd_table.py:56-89 does (approach is "" for the mask)."""
    for root, _, files in os.walk(_priorities(output_folder)):
        for file in files:
            if not file.endswith(".npy") or not file.startswith(f"{case_study}_{ds_name}"):
                continue
            arr = np.load(os.path.join(root, file))
            if file.endswith("is_misclassified.npy"):
                _, _, model_id, _, _ = file.split("_")
                yield MISCLASSIFIED, "", model_id, arr
            elif file.endswith("cam_order.npy"):
                if "dsa" in file or "lsa" in file:
                    _, _, model_id, metric, _, _ = file.split("_")
                    metric = approach_name(metric, cam=True)
                else:
                    _, _, model_id, metric, param, _, _ = file.split("_")
                    metric = approach_name(metric, param=param, cam=True)
                yield CAM_ORDER, metric, model_id, arr
            else:
                if "uncertainty" in file:
                    stem = file.replace(".npy", "").replace(f"{case_study}_{ds_name}_", "")
                    model_id, metric = stem.split("_uncertainty_")
                elif "dsa" in file or "lsa" in file:
                    _, _, model_id, metric, _ = file.split("_")
                else:
                    _, _, model_id, metric, param, _ = file.split("_")
                    metric = approach_name(metric, param=param, cam=False)
                yield SCORES, metric, model_id, arr


def order_from_scores(scores) -> np.ndarray:
    """eval_apfd_table.py:86: the highest score first, ties in `np.argsort`'s order."""
    return np.argsort(-np.asarray(scores))


def load_orders(output_folder: str, case_study: str, ds_name: str) -> Tuple[Dict[Tuple[str, str], np.ndarray], Dict[str, np.ndarray]]:
    """(orders[(approach, model_id)], misclassifications[model_id]) parsed from the file names exactly as
    eval_apfd_table.py:56-89 does."""
    misclassifications: Dict[str, np.ndarray] = {}
    orders: Dict[Tuple[str, str], np.ndarray] = {}
    for kind, approach, model_id, arr in _priority_files(output_folder, case_study, ds_name):
        if kind == MISCLASSIFIED:
            if int(model_id) < FIRST_K_MODELS_CONSIDERED:
                misclassifications[model_id] = arr
        else:
            orders[(approach, model_id)] = arr if kind == CAM_ORDER else order_from_scores(arr)
    return orders, misclassifications


def apfd_values(is_misclassified, scores: Dict[str, object], cam_orders: Dict[str, object]) -> Dict[str, float]:
    """{approach: APFD} of one model on one dataset, as eval_apfd_table.py:86-101 rates it: `scores[approach]` ranked
    by `order_from_scores`, `cam_orders[approach]` taken as stored, both against the misclassification mask."""
    mask = np.asarray(is_misclassified)
    res = {approach: apfd_from_order(mask, order_from_scores(s)) for approach, s in scores.items()}
    res.update({approach: apfd_from_order(mask, np.asarray(order)) for approach, order in cam_orders.items()})
    return res


def load_apfd_values(output_folder: str, case_study: str, ds_name: str) -> Dict[str, Dict[int, float]]:
    """APFD per approach and model id (eval_apfd_table.py:43-108; every approach found on disk is reported)."""
    mis: Dict[str, np.ndarray] = {}
    arrays: Dict[str, Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]] = {}
    for kind, approach, model_id, arr in _priority_files(output_folder, case_study, ds_name):
        if kind == MISCLASSIFIED:
            if int(model_id) < FIRST_K_MODELS_CONSIDERED:
                mis[model_id] = arr
        else:
            arrays.setdefault(model_id, ({}, {}))[kind == CAM_ORDER][approach] = arr
    apfds: Dict[str, Dict[int, float]] = {}
    for model_id, (scores, cam_orders) in arrays.items():
        if model_id not in mis:
            continue
        for approach, apfd in apfd_values(mis[model_id], scores, cam_orders).items():
            apfds.setdefault(approach, {})[int(model_id)] = apfd
    return apfds


# Table 1 of the study (src/plotters/eval_apfd_table.py, times_collector.py, utils.py)

TIME_COL = "time"                          # eval_apfd_table.py:23
CASE_STUDIES = ("mnist", "fmnist", "cifar10", "imdb")
N_FIRST_MODELS_TIMED = 10                  # times_collector.py:10

UNCERTAINTY_APPROACHES = ["deep_gini", "softmax", "pcs", "softmax_entropy", "VR"]
SURPRISE_APPROACHES = ["dsa", "pc-lsa", "pc-mdsa", "pc-mlsa", "pc-mmdsa"]
COVERAGE_APPROACHES = ["NAC_0.75", "NAC_0", "NBC_0.5", "NBC_0", "NBC_1", "SNAC_0.5", "SNAC_0", "SNAC_1", "TKNC_1",
                       "TKNC_2", "TKNC_3", "KMNC_2"]
# the table's rows, in the order of utils.py:21-61: every coverage and surprise TIP with its CAM row first
APPROACHES = ([a for c in COVERAGE_APPROACHES + SURPRISE_APPROACHES for a in (f"{c}-cam", c)]
              + UNCERTAINTY_APPROACHES)

# times_collector.py:23-28: the time files' renaming, applied in this order to the whole file name
_TIME_FILE_RENAMES = (("softmax_entropy", "SE"), ("pcs", "PCS"), ("deep_gini", "DeepGini"), ("softmax", "SM"))


def category(approach: str) -> Optional[str]:
    """utils.py:137-157: the table's row group of an approach (None for a name it does not know)."""
    if approach in UNCERTAINTY_APPROACHES:
        return "uncertainty"
    if approach in SURPRISE_APPROACHES or approach in [f"{a}-cam" for a in SURPRISE_APPROACHES]:
        return "surprise"
    if approach in ("original", "random"):
        return "baseline"
    if any(approach.startswith(nc) for nc in ("NAC", "NBC", "SNAC", "TKNC", "KMNC")):
        return "neuron coverage"
    return None


def _table_row(approach: str) -> Tuple[Optional[str], str]:
    return category(approach), approach


def load_time_files(output_folder: str) -> Dict[Tuple[str, str, str, str, str], List[float]]:
    """{(case_study, dataset, model_id, metric, param): [setup, pred, quant, cam]} of every time file of the models
    with ids below N_FIRST_MODELS_TIMED, keyed as times_collector.py:13-42 keys them (SE, PCS, DeepGini, SM for
    the uncertainty quantifiers; param "" for a metric without one)."""
    times = {}
    for root, _, files in os.walk(os.path.join(output_folder, "times")):
        for file in files:
            name = file
            for old, new in _TIME_FILE_RENAMES:
                name = name.replace(old, new)
            split = name.split("_")
            if len(split) == 5:
                key = tuple(split)
            elif len(split) == 4:
                key = tuple(split) + ("",)
            else:
                raise ValueError(f"{os.path.join(root, file)} is not named <case_study>_<dataset>_<model_id>_<metric>")
            if int(key[2]) >= N_FIRST_MODELS_TIMED:
                continue
            with open(os.path.join(root, file), "rb") as f:
                times[key] = pickle.load(f)
    return times


def _time_row(metric: str, param: str) -> Tuple[Optional[str], str]:
    """eval_apfd_table.py:235-243: a time file's (metric, param) as the table row it fills."""
    metric = {"SM": "softmax", "SE": "softmax_entropy", "PCS": "pcs", "DeepGini": "deep_gini"}.get(metric, metric)
    return _table_row(f"{metric}_{param}" if param != "" else metric)


def apfd_table(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES):
    """Table 1 of the study as the pandas DataFrame eval_apfd_table.py builds (`_fill_times(_get_as_df(...))`,
    :111-131, :176-249) from the result files under `output_folder`: rows (category, approach) in APPROACHES'
    order, columns (case study, "nominal" / "ood" / "time").

    An APFD cell is the mean of the approach's APFDs over the model ids below FIRST_K_MODELS_CONSIDERED, in
    ascending id order (`np.mean`), or "n.a." when no such model has it.  A time cell averages the time files of the
    model ids below N_FIRST_MODELS_TIMED over both datasets (`statistics.mean` per entry) as `setup + 2 * (pred +
    quant)`, plus `2 * cam` in a "-cam" row, formatted f"{round(t)}s".  A TIP that has time files in some case study
    but none in this one gets "n.a." in its row (and its "-cam" row); the reference allows this for VR on cifar10
    only, where the result is the same.  A TIP with no time file anywhere leaves its cells empty (NaN), and time files
    of case studies not in `case_studies` fill no cell.  ValueError when there is no time file of such a model."""
    import pandas as pd

    case_studies = list(case_studies)
    columns = pd.MultiIndex.from_product([case_studies, ["nominal", "ood", TIME_COL]])
    index = pd.MultiIndex.from_tuples([_table_row(a) for a in APPROACHES], names=["category", "approach"])
    df = pd.DataFrame(columns=columns, index=index)
    for case_study in case_studies:
        for ds in ("nominal", "ood"):
            apfds = load_apfd_values(output_folder, case_study, ds)
            for approach in APPROACHES:
                if approach in apfds:
                    per_model = apfds[approach]
                    value = np.mean([per_model[i] for i in sorted(per_model)])
                else:
                    value = "n.a."
                df.loc[_table_row(approach), (case_study, ds)] = value

    times = load_time_files(output_folder)
    if not times:
        raise ValueError(f"no time file of a model id below {N_FIRST_MODELS_TIMED} under {output_folder}")
    tips = sorted({(k[3], k[4]) for k in times})
    for case_study in case_studies:
        for metric, param in tips:
            row = _time_row(metric, param)
            cam_row = (row[0], f"{row[1]}-cam") if row[0] in ("surprise", "neuron coverage") else None
            entries = [v for k, v in times.items() if k[0] == case_study and k[3] == metric and k[4] == param]
            if not entries:
                for r in (row, cam_row):
                    if r is not None:
                        df.loc[r, (case_study, TIME_COL)] = "n.a."
                continue
            setup, pred, quant, cam = (statistics.mean(v[i] for v in entries) for i in range(4))
            non_cam = setup + 2 * (pred + quant)
            df.loc[row, (case_study, TIME_COL)] = f"{round(non_cam)}s"
            if cam_row is not None:
                df.loc[cam_row, (case_study, TIME_COL)] = f"{round(non_cam + 2 * cam)}s"
    return df


def write_apfd_table(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES) -> str:
    """`apfd_table(...)` as <output_folder>/results/apfds.csv (eval_apfd_table.py:252-257, the same bytes); the
    folder is created when missing.  Returns the file's path."""
    df = apfd_table(output_folder, case_studies)
    folder = os.path.join(output_folder, "results")
    os.makedirs(folder, exist_ok=True)
    path = os.path.join(folder, "apfds.csv")
    df.to_csv(path)
    return path
