"""Table 1 of the study (src/plotters/eval_apfd_table.py) from the UNMODIFIED reference (TEST INFRASTRUCTURE ONLY).

`write(folder)` builds a seeded synthetic result folder of the prioritization experiment, named and typed as
eval_prioritization.py:22-58 writes it.  Per case study and dataset it holds model ids on both sides of the table's
two cut-offs (APFDs of ids below 100, times of ids below 10), tied integer coverage scores, ties among the
uncertainties, VR missing on cifar10 (as for the study's dropout-free cifar10 model), no result at all for pc-mmdsa,
and no CAM order for TKNC_3.

`load_plotters(folder)` imports the reference's `src.plotters.{utils, times_collector, eval_apfd_table}` reading
`folder`.  They import only OUTPUT_FOLDER and DROPOUT_SAMPLE_SIZE from the TensorFlow-bound
`src.dnn_test_prio.case_study` and `handler_model`, so two stub modules carrying those stand in for them (the
other shims of oracle/ref_harness.py are not needed).  Usable only where the reference checkout exists.

    python oracle/apfd_table_oracle.py

writes tests/golden/apfd_table_reference.csv: the CSV the reference's `eval_apfd_table.run()` writes for
`write`'s folder, so that tests/test_apfd_table.py checks `results.write_apfd_table` where the checkout is absent.
"""
from __future__ import annotations

import importlib
import io
import os
import pickle
import shutil
import sys
import tempfile
import types
import warnings
from contextlib import redirect_stdout

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.ref_harness import REFERENCE_ROOT, available  # noqa: E402

GOLDEN_CSV = os.path.join(ROOT, "tests", "golden", "apfd_table_reference.csv")

CASE_STUDIES = ("mnist", "fmnist", "cifar10", "imdb")
MODEL_IDS = (0, 1, 2, 3, 7, 12, 99, 100, 140)
UNCERTAINTIES = ("softmax", "pcs", "softmax_entropy", "deep_gini", "VR")
NC_METRICS = ("NBC_0", "NBC_0.5", "NBC_1", "SNAC_0", "SNAC_0.5", "SNAC_1", "NAC_0", "NAC_0.75", "TKNC_1", "TKNC_2",
              "TKNC_3", "KMNC_2")
SAS = ("dsa", "pc-lsa", "pc-mdsa", "pc-mlsa")      # pc-mmdsa is missing altogether
NO_CAM_ORDER = ("TKNC_3",)
SEED = 20261017


def _save(folder, name, arr):
    np.save(os.path.join(folder, "priorities", f"{name}.npy"), arr)


def _times(folder, name, values):
    with open(os.path.join(folder, "times", name), "wb") as f:
        pickle.dump(values, f)


def write(folder: str, seed: int = SEED) -> str:
    """Writes the folder's priorities/ and times/ under `folder` (created when missing); returns `folder`."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(folder, "priorities"), exist_ok=True)
    os.makedirs(os.path.join(folder, "times"), exist_ok=True)
    for cs_i, cs in enumerate(CASE_STUDIES):
        n = 40 + 7 * cs_i
        for ds in ("nominal", "ood"):
            for model_id in MODEL_IDS:
                stem = f"{cs}_{ds}_{model_id}"
                mask = rng.random(n) < 0.3
                mask[rng.integers(n)] = True
                _save(folder, f"{stem}_is_misclassified", mask)
                for q in UNCERTAINTIES:
                    if q == "VR" and cs == "cifar10":
                        continue
                    # few distinct values: ties that np.argsort must break
                    _save(folder, f"{stem}_uncertainty_{q}", rng.integers(0, 6, n).astype(np.float64) / 5)
                    _times(folder, f"{stem}_{q}", [0, float(rng.uniform(0, 30)), float(rng.uniform(0, 3)), 0])
                for metric in NC_METRICS:
                    _save(folder, f"{stem}_{metric}_scores", rng.integers(0, 4, n).astype(np.int32))
                    if metric not in NO_CAM_ORDER:
                        _save(folder, f"{stem}_{metric}_cam_order", rng.permutation(n).astype(np.int64))
                    _times(folder, f"{stem}_{metric}", [float(v) for v in rng.uniform(0, 40, 4)])
                for sa in SAS:
                    _save(folder, f"{stem}_{sa}_scores", np.round(rng.random(n) * 4) / 4)
                    _save(folder, f"{stem}_{sa}_cam_order", rng.permutation(n).astype(np.int64))
                    _times(folder, f"{stem}_{sa}", [float(v) for v in rng.uniform(0, 90, 4)])
    return folder


def load_plotters(output_folder: str) -> types.SimpleNamespace:
    """The reference's `src.plotters.{utils, times_collector, eval_apfd_table}` (unmodified) reading `output_folder`:
    the stub `src.dnn_test_prio.case_study` carries OUTPUT_FOLDER = `output_folder` + "/" (eval_apfd_table.py:257
    appends "results/" to it without a slash), the stub `src.dnn_test_prio.handler_model` DROPOUT_SAMPLE_SIZE.
    Imported afresh on every call, so each namespace reads its own folder."""
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
        # the reference must win `import src...`: this repository's own src/ overlay leaves the path meanwhile
        here = os.path.abspath(ROOT)
        sys.path[:] = [REFERENCE_ROOT] + [p for p in saved_path if os.path.abspath(p or ".") != here]
        importlib.invalidate_caches()
        sys.modules[case_study.__name__] = case_study
        sys.modules[handler_model.__name__] = handler_model
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SyntaxWarning)                    # eval_apfd_table.py:159 "\m"
            mods = {name: importlib.import_module(f"src.plotters.{name}")
                    for name in ("utils", "times_collector", "eval_apfd_table")}
        for mod in list(mods.values()) + [sys.modules["src.core.apfd"]]:
            assert os.path.abspath(mod.__file__).startswith(os.path.abspath(REFERENCE_ROOT)), mod.__file__
        return types.SimpleNamespace(**mods)
    finally:
        sys.path[:] = saved_path
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        sys.modules.update(saved_src)


def reference_table(output_folder: str, case_studies=("mnist", "fmnist", "cifar10", "imdb")):
    """eval_apfd_table.py's `_fill_times(_get_as_df(case_studies))` over `output_folder`, its progress lines and
    missing-result warnings silenced."""
    ref = load_plotters(output_folder)
    with redirect_stdout(io.StringIO()), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return ref.eval_apfd_table._fill_times(ref.eval_apfd_table._get_as_df(list(case_studies)))


def reference_csv(output_folder: str) -> bytes:
    """The bytes of the results/apfds.csv the reference's `eval_apfd_table.run()` writes for `output_folder`
    (run on a copy of the folder, so `output_folder` is left as it was).  run() goes on to the LaTeX table
    (`_plot_latex_table`) after writing the CSV; that file is not read here."""
    with tempfile.TemporaryDirectory() as tmp:
        copy = os.path.join(tmp, "out")
        shutil.copytree(output_folder, copy)
        os.makedirs(os.path.join(copy, "results"))
        ref = load_plotters(copy)
        with redirect_stdout(io.StringIO()), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref.eval_apfd_table.run()
        with open(os.path.join(copy, "results", "apfds.csv"), "rb") as f:
            return f.read()


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        csv = reference_csv(write(os.path.join(tmp, "out")))
    with open(GOLDEN_CSV, "wb") as f:
        f.write(csv)
    print(GOLDEN_CSV, len(csv), "bytes")
