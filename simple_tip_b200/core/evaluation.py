"""The study's evaluation phase (reproduction.py `--phase evaluation`, its four `EvalType`s) without TensorFlow.

Table 2 (`active_learning_table`, src/plotters/eval_active_learning_table.py) is built from the pickles
`active_learning.evaluate` leaves in `<out>/active_learning/`; the Wilcoxon signed-rank p-values and paired
Vargha-Delaney effect sizes between every two approaches (`apfd_statistics`, eval_apfd_correlation.py;
`active_learning_statistics`, eval_active_correlation.py) from those pickles and from the APFDs of
`<out>/priorities/`.  `evaluate_results` writes what one evaluation type of the reference writes under
`<out>/results/`, minus its LaTeX tables and heatmap PNGs.  The reference's scripts need TensorFlow (through
`case_study`) and pingouin; these need pandas and scipy only, imported inside the functions that use them.

The reference's quirks are kept, so the files come out with the same bytes: its file-name regexes, the order its
means sum in, and the statistics' keys, which carry the case study but not the dataset (DESIGN.md §9).
Host-side only.
"""
from __future__ import annotations

import os
import pickle
import re
import warnings
from typing import Dict, List, Mapping, Sequence, Set, Tuple

import numpy as np

from .results import APPROACHES, CASE_STUDIES, category, load_apfd_values, write_apfd_table

BASELINE = "random"                        # eval_active_learning_table.py:19
ORIGINAL = "original"
NUM_RUNS = 100                             # utils.py:11
SPLITS = ("nominal", "ood")
# reproduction.py:29-35 (`EvalType`)
EVAL_TYPES = ("test_prio", "active_learning", "test_prio_statistics", "active_learning_statistics")

# the fill values of calc_values' grids (correlation_plot.py:71-86): what a pair i >= j keeps
P_FILL, E_FILL, NUM_SAMPLES_FILL = 10000, -10000, -1000

RunResult = Dict[Tuple[str, str], float]
"""{("nominal" / "ood", "observed" / "future"): accuracy}, one pickle of `results.persist_active_learning`"""


def human_approach_name(approach: str) -> str:
    """utils.py:100-113: the approach's name in the paper ("NAC_0.75-cam" -> "NAC-0.75-CAM")."""
    names = {"softmax_entropy": "Entropy", "VR": "MC-Dropout", "softmax": "Vanilla SM", "deep_gini": "DeepGini"}
    if approach in names:
        return names[approach]
    if approach in ("uncertainty", "surprise", "neuron coverage", "baseline"):
        return approach
    return approach.replace("_", "-").upper()


# Table 2 (src/plotters/eval_active_learning_table.py)

def load_active_learning(output_folder: str, case_study: str, ds_name: str, by_id: bool = False) -> Dict[str, object]:
    """eval_active_learning_table.py:26-59: {approach: [run results]} (by_id: {approach: {model id: run result}})
    for every approach of APPROACHES, `random` and `original`, in that order.

    A file belongs to an approach when `re.match(f"{case_study}_\\d*_{approach}_{ds_name}\\.", name)` holds
    (`original`: `f"{case_study}_\\d*_original_na\\."`), unescaped as in the reference: the "." of NAC_0.75 matches
    any character.  Files are taken in `os.walk` order over `<out>/active_learning`, and read from that folder
    itself even when found in a subfolder (utils.py:168-184), so a subfolder file counts once more for the
    top-level file of its name.  The model id is the name's second "_" field."""
    folder = os.path.join(output_folder, "active_learning")
    names = [file for _, _, files in os.walk(folder) for file in files]
    patterns = [(a, f"{case_study}_\\d*_{a}_{ds_name}\\.") for a in APPROACHES + [BASELINE]]
    patterns.append((ORIGINAL, f"{case_study}_\\d*_original_na\\."))
    res: Dict[str, object] = {}
    for approach, pattern in patterns:
        regex = re.compile(pattern)
        matches = [name for name in names if regex.match(name, pos=0)]
        runs = []
        for name in matches:
            with open(os.path.join(folder, name), "rb") as f:
                runs.append(pickle.load(f))
        res[approach] = {int(n.split("_")[1]): r for n, r in zip(matches, runs)} if by_id else runs
    return res


def _reduce_active_learning(case_study: str, runs_by_approach: Mapping[str, List[RunResult]]) -> Dict[str, RunResult]:
    """eval_active_learning_table.py:62-84: each approach's mean over its runs, Python's `sum(...) / len(...)` in the
    loader's order; an approach without runs is left out, with a warning unless it is VR on cifar10."""
    res = {}
    for approach, runs in runs_by_approach.items():
        assert all(runs[0].keys() == runs[i].keys() for i in range(1, len(runs)))
        if len(runs) == 0:
            if not (approach == "VR" and case_study == "cifar10"):
                warnings.warn("missing results")
            continue
        res[approach] = {key: sum(run[key] for run in runs) / len(runs) for key in runs[0]}
    return res


def _relative_gains(reduced: Mapping[str, RunResult]) -> Dict[str, RunResult]:
    """eval_active_learning_table.py:87-100: every approach's mean minus the `random` baseline's."""
    assert BASELINE in reduced.keys()
    return {approach: {key: perf[key] - reduced[BASELINE][key] for key in perf}
            for approach, perf in reduced.items() if approach != BASELINE}


def active_learning_table(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES):
    """Table 2 of the study as the pandas DataFrame eval_active_learning_table.py:103-151 (`build_data_frame`)
    builds: rows (category, approach) for `original`, `random` and APPROACHES; columns (case study, active split
    "nominal" / "ood", "<evaluation split>:observed" / ":future").

    `original` and `random` show their mean accuracies, every TIP its mean minus `random`'s, as "{:.2%}" strings.  A
    TIP without runs gets "n.a."; a cell no run names stays NaN.  AssertionError when a (case study, active split)
    has no `random` run or runs with differing keys, KeyError when it has no `original` run."""
    import pandas as pd

    case_studies = list(case_studies)
    eval_splits = [f"{ds}:{part}" for ds in SPLITS for part in ("observed", "future")]
    columns = pd.MultiIndex.from_product([case_studies, list(SPLITS), eval_splits])
    rows = [(category(a), a) for a in [ORIGINAL, BASELINE] + APPROACHES]
    df = pd.DataFrame(columns=columns, index=pd.MultiIndex.from_tuples(rows, names=["category", "approach"]))
    for cs in case_studies:
        for active_split in SPLITS:
            reduced = _reduce_active_learning(cs, load_active_learning(output_folder, cs, active_split))
            relative = _relative_gains(reduced)
            for approach in (ORIGINAL, BASELINE):
                for key, value in reduced[approach].items():
                    df.at[(category(approach), approach), (cs, active_split, f"{key[0]}:{key[1]}")] = f"{value:.2%}"
            for approach in APPROACHES:
                row = (category(approach), approach)
                if approach not in relative:
                    for split in eval_splits:
                        df.at[row, (cs, active_split, split)] = "n.a."
                    continue
                for key, value in relative[approach].items():
                    df.at[row, (cs, active_split, f"{key[0]}:{key[1]}")] = f"{value:.2%}"
    return df


def _results_path(output_folder: str, name: str) -> str:
    folder = os.path.join(output_folder, "results")
    os.makedirs(folder, exist_ok=True)
    return os.path.join(folder, name)


def write_active_learning_table(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES) -> str:
    """`active_learning_table(...)` as <output_folder>/results/active.csv (eval_active_learning_table.py:227-231, the
    same bytes); the folder is created when missing.  Returns the file's path."""
    df = active_learning_table(output_folder, case_studies)
    path = _results_path(output_folder, "active.csv")
    df.to_csv(path)
    return path


# The statistics (src/plotters/correlation_plot.py, eval_apfd_correlation.py, eval_active_correlation.py)

def wilcoxon_p(x: Sequence[float], y: Sequence[float]) -> float:
    """The two-sided p-value of the Wilcoxon signed-rank test of the pairs (x[i], y[i]), as pingouin 0.5.0's
    `wilcoxon(x, y, alternative="two-sided")` gets it from scipy 1.4.1: zero differences dropped
    (zero_method="wilcox"), average ranks of |x - y|, the normal approximation with the tie-corrected variance, no
    continuity correction.  For the same n, T and ties the float operations are scipy 1.4.1's, so the bits are too.
    Newer scipy versions may take the exact distribution instead when at most 50 non-zero differences remain (the
    limit and the handling of ties depend on the version); the study's pairs have hundreds.  ValueError when every
    difference is zero, as in scipy."""
    from scipy.special import ndtr

    d = np.asarray(x, dtype=np.float64) - np.asarray(y, dtype=np.float64)
    if np.all(d == 0):
        raise ValueError("the Wilcoxon test needs at least one pair whose values differ")
    d = d[d != 0]
    n = d.size
    _, group, counts = np.unique(np.abs(d), return_inverse=True, return_counts=True)
    # a tie group holding ranks last - count + 1 .. last has the average rank last - (count - 1) / 2
    ranks = (np.cumsum(counts) - (counts - 1) / 2)[group]
    r_plus, r_minus = np.sum((d > 0) * ranks), np.sum((d < 0) * ranks)
    mn = n * (n + 1.0) * 0.25
    se = n * (n + 1.0) * (2.0 * n + 1.0)
    ties = counts[counts > 1]
    if ties.size:
        se -= 0.5 * (ties * (ties * ties - 1)).sum()
    z = (min(r_plus, r_minus) - mn) / np.sqrt(se / 24)
    return float(2.0 * ndtr(-abs(z)))


def paired_a12(x: Sequence[float], y: Sequence[float]) -> float:
    """correlation_plot.py:20-30 (`_paired_vargha_delanay_a12`): 2 * |(#(x > y) + #(x == y) / 2) / n - 1/2|, from 0
    (either side as likely) to 1 (one side always greater)."""
    x, y = np.asarray(x), np.asarray(y)
    assert x.shape == y.shape
    a12 = (np.sum(x > y) + 0.5 * np.sum(x == y)) / x.size
    return float(2 * abs(a12 - 0.5))


def wilcoxon_a12(measurements: Mapping[str, Mapping[str, float]], approaches: Sequence[str]) -> Dict[str, np.ndarray]:
    """correlation_plot.py:69-101 (`WilcoxonCorrelationPlot.calc_values`): {"p", "e", "num_samples"} grids over
    `approaches`, of which only the upper triangle i < j is computed.  A pair is compared on the samples (keys of
    `measurements[approach]`) both approaches have: NaN in "p" and "e" when they share none or their values are
    equal, otherwise `wilcoxon_p` and `paired_a12`.  The other cells keep P_FILL, E_FILL and NUM_SAMPLES_FILL.
    Measurements of approaches not in `approaches` are ignored."""
    size = (len(approaches), len(approaches))
    res = {"p": np.full(size, P_FILL, dtype=np.float64), "e": np.full(size, E_FILL, dtype=np.float64),
           "num_samples": np.full(size, NUM_SAMPLES_FILL, dtype=np.int64)}
    for i in range(len(approaches) - 1):
        mi = measurements.get(approaches[i], {})
        for j in range(i + 1, len(approaches)):
            mj = measurements.get(approaches[j], {})
            keys = set(mi).intersection(mj)
            xi, xj = [mi[k] for k in keys], [mj[k] for k in keys]
            res["num_samples"][i, j] = len(keys)
            if len(keys) == 0 or xi == xj:
                res["p"][i, j] = res["e"][i, j] = np.nan
            else:
                res["p"][i, j], res["e"][i, j] = wilcoxon_p(xi, xj), paired_a12(xi, xj)
    return res


def _missing_runs(values: Mapping[str, Mapping[int, float]], has_dropout: bool) -> Set[int]:
    """utils.py:187-201 (`identify_incomplete_values`): the run ids below NUM_RUNS some approach has no value of (VR
    counts only for a model with dropout)."""
    return {i for approach, runs in values.items() for i in range(NUM_RUNS)
            if i not in runs and (approach != "VR" or has_dropout)}


def _by_case_study_and_run(per_split: Sequence[Tuple[str, Mapping[str, Mapping[int, float]]]]
                           ) -> Dict[str, Dict[str, float]]:
    """utils.py:204-229 (`named_tuples`) per (case study, dataset) in the given order, flattened with `dict.update` as
    eval_apfd_correlation.py:49-55 does: {approach: {f"{case_study}_{model id}": value}}.  The key names no dataset,
    so a later dataset's value of a model replaces the earlier one's."""
    res: Dict[str, Dict[str, float]] = {}
    for cs, values in per_split:
        for approach, runs in values.items():
            res.setdefault(approach, {}).update({f"{cs}_{run_id}": v for run_id, v in runs.items()})
    return res


Statistics = Tuple[Dict[str, np.ndarray], Dict[Tuple[str, str], Set[int]]]
"""(`wilcoxon_a12` grids over APPROACHES, {(case study, dataset): missing run ids})"""


def apfd_statistics(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES) -> Statistics:
    """eval_apfd_correlation.py:27-103 without the heatmap: every approach's APFDs of the model ids below
    FIRST_K_MODELS_CONSIDERED (`results.load_apfd_values`), one sample per case study and model, compared pairwise by
    `wilcoxon_a12`.  Since a sample's key names no dataset, a model's OOD APFD replaces its nominal one, as in the
    reference: the statistics compare OOD APFDs (and nominal ones of models without OOD results)."""
    per_split, missing = [], {}
    for cs in case_studies:
        for ds in SPLITS:
            values = {a: v for a, v in load_apfd_values(output_folder, cs, ds).items() if a in APPROACHES}
            missing[cs, ds] = _missing_runs(values, has_dropout=cs != "cifar10")
            per_split.append((cs, values))
    return wilcoxon_a12(_by_case_study_and_run(per_split), APPROACHES), missing


def active_learning_statistics(output_folder: str, case_studies: Sequence[str] = CASE_STUDIES) -> Statistics:
    """eval_active_correlation.py:48-117 without the heatmap: every retrained model's accuracy on the future split of
    the dataset it was selected from, for the model ids below NUM_RUNS, compared pairwise by `wilcoxon_a12` with the
    same keys as `apfd_statistics` (so a model's OOD-selected value replaces its nominal one).  `original` and
    `random` count for the missing runs but are not compared."""
    per_split, missing = [], {}
    for cs in case_studies:
        for ds in SPLITS:
            loaded = load_active_learning(output_folder, cs, ds, by_id=True)
            values = {a: {} for a in APPROACHES + [ORIGINAL, BASELINE]}
            for i in range(NUM_RUNS):
                for approach, runs in loaded.items():
                    if i in runs:
                        values[approach][i] = runs[i][(ds, "future")]
            missing[cs, ds] = _missing_runs(values, has_dropout=cs != "cifar10")
            per_split.append((cs, values))
    return wilcoxon_a12(_by_case_study_and_run(per_split), APPROACHES), missing


def statistics_frames(grids: Mapping[str, np.ndarray]):
    """(p, e) DataFrames as eval_apfd_correlation.py:84-101 writes them, indexed both ways by the approaches' paper
    names.  P_FILL becomes "" in the p frame only; the reference's second `replace` also goes to the p frame, so the
    e frame keeps E_FILL."""
    import pandas as pd

    names = [human_approach_name(a) for a in APPROACHES]
    p = pd.DataFrame(data=grids["p"], index=names, columns=names).replace(P_FILL, "")
    return p, pd.DataFrame(data=grids["e"], index=names, columns=names)


def write_statistics(output_folder: str, experiment: str, grids: Mapping[str, np.ndarray]) -> Tuple[str, str]:
    """`statistics_frames(grids)` as <output_folder>/results/<experiment>_correlation_p.csv and _eff.csv, the
    reference's file names for experiment "apfd" and "active"; the folder is created when missing.  Returns the two
    paths."""
    p, e = statistics_frames(grids)
    paths = (_results_path(output_folder, f"{experiment}_correlation_p.csv"),
             _results_path(output_folder, f"{experiment}_correlation_eff.csv"))
    p.to_csv(paths[0])
    e.to_csv(paths[1])
    return paths


def evaluate_results(output_folder: str, eval_type: str, case_studies: Sequence[str] = CASE_STUDIES) -> List[str]:
    """reproduction.py --phase evaluation for one `EvalType` value: the CSVs its script writes under
    <output_folder>/results/ ("test_prio": apfds.csv, "active_learning": active.csv, "test_prio_statistics":
    apfd_correlation_{p,eff}.csv, "active_learning_statistics": active_correlation_{p,eff}.csv), without the LaTeX
    tables and heatmaps.  The statistics warn with the runs some approach misses, per case study and dataset, where
    the reference prints them.  Returns the paths written; ValueError for another `eval_type`."""
    if eval_type == "test_prio":
        return [write_apfd_table(output_folder, case_studies)]
    if eval_type == "active_learning":
        return [write_active_learning_table(output_folder, case_studies)]
    if eval_type == "test_prio_statistics":
        experiment, (grids, missing) = "apfd", apfd_statistics(output_folder, case_studies)
    elif eval_type == "active_learning_statistics":
        experiment, (grids, missing) = "active", active_learning_statistics(output_folder, case_studies)
    else:
        raise ValueError(f"unknown evaluation type {eval_type!r}; expected one of {EVAL_TYPES}")
    for (cs, ds), runs in missing.items():
        if runs:
            warnings.warn(f"Missing values {cs} - {ds}: {sorted(runs)}")
    return list(write_statistics(output_folder, experiment, grids))
