"""Table 2 and the statistics of the study (src/plotters/eval_active_learning_table.py, eval_apfd_correlation.py,
eval_active_correlation.py) from the UNMODIFIED reference (TEST INFRASTRUCTURE ONLY).

`write(folder)` builds a seeded synthetic result folder: the prioritization results of
oracle/apfd_table_oracle.py under priorities/ and times/, and the active-learning experiment's pickles under
active_learning/, named and keyed as eval_active_learning.py:134-147 writes them.  Per case study the latter hold
model ids on both sides of the statistics' cut-off of 100, accuracies k / 50 (so differences tie), no VR on cifar10,
no TKNC_3-cam for the nominal split of mnist, no KMNC_2 for the OOD split of fmnist, SNAC_1 equal to SNAC_0
(identical samples), pc-mmdsa-cam and pc-mmdsa of disjoint models (no shared sample), the NAC_0.75 files of one model
named NAC_0x75 (the regexes' unescaped ".") and, in a subfolder, a differing copy of one file (which the reference
reads from the top-level folder instead).

`load_plotters(folder)` imports the reference's three scripts reading `folder`.  Besides the `case_study` /
`handler_model` stubs of apfd_table_oracle.py, correlation_plot.py needs pingouin, matplotlib and seaborn, none of
which is installed here: stubs stand in for them during the import and `run()` only.  pingouin's stub computes
`wilcoxon(...)["p-val"][0]` with `scipy141_wilcoxon_p`, a restatement of the code path pingouin 0.5.0 takes through
scipy 1.4.1's `wilcoxon`; the plotting stubs accept any call and draw nothing.  `calc_values` also needs NumPy's
removed `np.float` / `np.int` aliases, set while `run()` runs.  Usable only where the reference checkout exists.

    python oracle/evaluation_oracle.py

writes the reference's results/active.csv and its four statistics CSVs for `write`'s folder to tests/golden/, so
that tests/test_evaluation.py checks `core.evaluation` where the checkout is absent.
"""
from __future__ import annotations

import contextlib
import importlib
import io
import os
import pickle
import shutil
import sys
import tempfile
import types
import warnings

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import apfd_table_oracle  # noqa: E402
from oracle.ref_harness import REFERENCE_ROOT, available  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
# results/<name> the reference writes -> its golden copy
GOLDEN = {name: os.path.join(GOLDEN_DIR, name.replace(".csv", "_reference.csv"))
          for name in ("active.csv", "apfd_correlation_p.csv", "apfd_correlation_eff.csv", "active_correlation_p.csv",
                       "active_correlation_eff.csv")}
# the reference's scripts, by the evaluation type that runs them (reproduction.py:67-82)
SCRIPTS = {"active_learning": "eval_active_learning_table", "test_prio_statistics": "eval_apfd_correlation",
           "active_learning_statistics": "eval_active_correlation"}

CASE_STUDIES = apfd_table_oracle.CASE_STUDIES
MODEL_IDS = (0, 1, 2, 5, 9, 23, 99, 100, 131)
SPLITS = ("nominal", "ood")
SPLIT_KEYS = [(ds, part) for ds in SPLITS for part in ("observed", "future")]
APPROACHES = ([f"{a}{cam}" for a in apfd_table_oracle.NC_METRICS + apfd_table_oracle.SAS + ("pc-mmdsa",)
               for cam in ("-cam", "")] + list(apfd_table_oracle.UNCERTAINTIES))
MISSING = {("mnist", "nominal", "TKNC_3-cam"), ("fmnist", "ood", "KMNC_2")}
ONLY_MODEL = {"pc-mmdsa-cam": 0, "pc-mmdsa": 1}
SUBFOLDER_COPY = "mnist_2_dsa_nominal.pickle"
SEED = 20261018


def _pickle(path, obj):
    with open(path, "wb") as f:
        pickle.dump(obj, f)


def write(folder: str, seed: int = SEED) -> str:
    """Writes the folder's priorities/, times/ and active_learning/ under `folder` (created when missing); returns
    `folder`."""
    apfd_table_oracle.write(folder)
    rng = np.random.default_rng(seed)
    al = os.path.join(folder, "active_learning")
    os.makedirs(os.path.join(al, "old"), exist_ok=True)

    def accuracies():
        return {key: int(rng.integers(20, 50)) / 50 for key in SPLIT_KEYS}

    for cs in CASE_STUDIES:
        for model_id in MODEL_IDS:
            _pickle(os.path.join(al, f"{cs}_{model_id}_original_na.pickle"), accuracies())
            for ds in SPLITS:
                for approach in APPROACHES + ["random"]:
                    if ((cs, ds, approach) in MISSING or (approach == "VR" and cs == "cifar10")
                            or ONLY_MODEL.get(approach, model_id) != model_id):
                        continue
                    name = "NAC_0x75" if approach == "NAC_0.75" and model_id == 5 else approach
                    if approach == "SNAC_1":
                        with open(os.path.join(al, f"{cs}_{model_id}_SNAC_0_{ds}.pickle"), "rb") as f:
                            res = pickle.load(f)
                    else:
                        res = accuracies()
                    _pickle(os.path.join(al, f"{cs}_{model_id}_{name}_{ds}.pickle"), res)
    _pickle(os.path.join(al, "old", SUBFOLDER_COPY), accuracies())
    return folder


def scipy141_wilcoxon_p(x, y) -> float:
    """`pingouin.wilcoxon(x, y, alternative="two-sided")["p-val"][0]` of pingouin 0.5.0 over scipy 1.4.1 (for inputs
    without NaN): scipy.stats.wilcoxon(x, y, zero_method="wilcox", correction=False, alternative="two-sided"), whose
    1.4.1 code always takes the normal approximation — zero differences dropped, `rankdata` of |d|, T the smaller
    rank sum, the variance less half the sum of t^3 - t over the repeated ranks, 2 * norm.sf(|z|)."""
    from scipy import stats

    d = np.asarray(x, dtype=np.float64) - np.asarray(y, dtype=np.float64)
    d = np.compress(np.not_equal(d, 0), d)
    count = len(d)
    r = stats.rankdata(abs(d))
    r_plus, r_minus = np.sum((d > 0) * r, axis=0), np.sum((d < 0) * r, axis=0)
    T = min(r_plus, r_minus)
    mn = count * (count + 1.) * 0.25
    se = count * (count + 1.) * (2. * count + 1.)
    repnum = np.unique(r, return_counts=True)[1]
    repnum = repnum[repnum > 1]
    if repnum.size != 0:
        se -= 0.5 * (repnum * (repnum * repnum - 1)).sum()
    se = np.sqrt(se / 24)
    z = (T - mn) / se
    return float(2. * stats.norm.sf(abs(z)))


class _Anything:
    """Stands for any matplotlib / seaborn object: every attribute and call gives itself, and it unpacks to
    nothing."""

    def __getattr__(self, name):
        return self

    def __call__(self, *args, **kwargs):
        return self

    def __iter__(self):
        return iter(())


def _stub_modules():
    anything = _Anything()
    mods = {}
    for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.colors", "seaborn"):
        mods[name] = types.ModuleType(name)
        mods[name].__getattr__ = lambda attr: anything
    mods["pingouin"] = types.ModuleType("pingouin")
    mods["pingouin"].wilcoxon = lambda x, y, alternative: {"p-val": [scipy141_wilcoxon_p(x, y)]}
    return mods


@contextlib.contextmanager
def _stubs():
    """The plotting / statistics stubs and NumPy's `float` / `int` aliases, in place for the block only."""
    stubs = _stub_modules()
    saved = {k: sys.modules[k] for k in stubs if k in sys.modules}
    aliases = {k: getattr(np, k) for k in ("float", "int") if k in np.__dict__}
    sys.modules.update(stubs)
    np.float, np.int = float, int
    try:
        yield
    finally:
        for k in stubs:
            del sys.modules[k]
        sys.modules.update(saved)
        for k in ("float", "int"):
            if k in aliases:
                setattr(np, k, aliases[k])
            else:
                delattr(np, k)


def load_plotters(output_folder: str) -> types.SimpleNamespace:
    """The reference's `src.plotters.{utils, correlation_plot, eval_active_learning_table, eval_apfd_correlation,
    eval_active_correlation}` (unmodified) reading `output_folder`, imported afresh as
    apfd_table_oracle.load_plotters imports its modules.  Call their functions inside `_stubs()`."""
    if not available():
        raise RuntimeError(f"reference not found under {REFERENCE_ROOT}")
    case_study = types.ModuleType("src.dnn_test_prio.case_study")
    case_study.OUTPUT_FOLDER = os.path.join(output_folder, "")
    handler_model = types.ModuleType("src.dnn_test_prio.handler_model")
    handler_model.DROPOUT_SAMPLE_SIZE = 200                                   # handler_model.py:7
    saved_path = list(sys.path)
    saved_src = {k: v for k, v in sys.modules.items() if k == "src" or k.startswith("src.")}
    for k in saved_src:
        del sys.modules[k]
    try:
        here = os.path.abspath(ROOT)
        sys.path[:] = [REFERENCE_ROOT] + [p for p in saved_path if os.path.abspath(p or ".") != here]
        importlib.invalidate_caches()
        sys.modules[case_study.__name__] = case_study
        sys.modules[handler_model.__name__] = handler_model
        with warnings.catch_warnings(), _stubs():
            warnings.simplefilter("ignore", SyntaxWarning)                    # the scripts' "\d", "\m"
            mods = {name: importlib.import_module(f"src.plotters.{name}")
                    for name in ["utils", "correlation_plot"] + list(SCRIPTS.values())}
        for mod in mods.values():
            assert os.path.abspath(mod.__file__).startswith(os.path.abspath(REFERENCE_ROOT)), mod.__file__
        return types.SimpleNamespace(**mods)
    finally:
        sys.path[:] = saved_path
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        sys.modules.update(saved_src)


def reference_table(output_folder: str, case_studies=CASE_STUDIES):
    """eval_active_learning_table.py's `build_data_frame(case_studies)` over `output_folder`, its progress lines
    and warnings silenced."""
    ref = load_plotters(output_folder)
    with contextlib.redirect_stdout(io.StringIO()), warnings.catch_warnings(), _stubs():
        warnings.simplefilter("ignore")
        return ref.eval_active_learning_table.build_data_frame(list(case_studies))


def reference_run(output_folder: str, eval_type: str):
    """Runs the reference's `run()` for `eval_type` on a copy of `output_folder` (left as it was).  Returns
    ({file name: bytes} of the CSVs it wrote to results/, the grids of its last `calc_values` — the full one over
    APPROACHES — or None for the table)."""
    with tempfile.TemporaryDirectory() as tmp:
        copy = os.path.join(tmp, "out")
        shutil.copytree(output_folder, copy)
        os.makedirs(os.path.join(copy, "results"))
        os.makedirs(os.path.join(copy, ".tmp"))             # the statistics' value cache
        ref = load_plotters(copy)
        grids = []
        plot = ref.correlation_plot.WilcoxonCorrelationPlot
        calc_values = plot.calc_values
        plot.calc_values = lambda self: grids.append(calc_values(self)) or grids[-1]
        with contextlib.redirect_stdout(io.StringIO()), warnings.catch_warnings(), _stubs():
            warnings.simplefilter("ignore")
            getattr(ref, SCRIPTS[eval_type]).run()
        files = {}
        for name in sorted(os.listdir(os.path.join(copy, "results"))):
            if name.endswith(".csv"):
                with open(os.path.join(copy, "results", name), "rb") as f:
                    files[name] = f.read()
        return files, (grids[-1] if grids else None)


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        folder = write(os.path.join(tmp, "out"))
        for eval_type in SCRIPTS:
            for name, data in reference_run(folder, eval_type)[0].items():
                with open(GOLDEN[name], "wb") as f:
                    f.write(data)
                print(GOLDEN[name], len(data), "bytes")
