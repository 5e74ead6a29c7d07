"""Table 1 of the study (results.apfd_table / write_apfd_table) against the reference's
src/plotters/eval_apfd_table.py on a seeded synthetic result folder (oracle/apfd_table_oracle.py): the DataFrame
against the reference's `_fill_times(_get_as_df(...))` where the reference checkout exists, the CSV against the one
its `run()` wrote (tests/golden/apfd_table_reference.csv) everywhere, and the two documented deviations."""
import os
import pickle
import shutil

import numpy as np
import pytest

pytest.importorskip("pandas")

from oracle import apfd_table_oracle as O      # noqa: E402
from oracle import ref_harness                 # noqa: E402
from simple_tip_b200.core import results as R  # noqa: E402


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    return O.write(str(tmp_path_factory.mktemp("results") / "out"))


def test_csv_equals_the_references_byte_for_byte(folder, tmp_path):
    out = str(tmp_path / "out")
    shutil.copytree(folder, out)
    path = R.write_apfd_table(out)
    assert path == os.path.join(out, "results", "apfds.csv")
    with open(path, "rb") as f, open(O.GOLDEN_CSV, "rb") as g:
        assert f.read() == g.read()


def test_table_equals_the_references_dataframe(folder):
    if not ref_harness.available():
        pytest.skip("the reference checkout is not available")
    mine, ref = R.apfd_table(folder), O.reference_table(folder)
    assert mine.index.equals(ref.index) and mine.columns.equals(ref.columns)
    assert mine.equals(ref)
    assert O.reference_csv(folder) == open(O.GOLDEN_CSV, "rb").read()


def test_cells(folder):
    df = R.apfd_table(folder)
    assert list(df.index) == [(R.category(a), a) for a in R.APPROACHES]
    # APFDs: the mean over the model ids below 100, in id order
    apfds = R.load_apfd_values(folder, "imdb", "ood")
    assert set(apfds["dsa"]) == {i for i in O.MODEL_IDS if i < 100}
    assert df.loc[("surprise", "dsa"), ("imdb", "ood")] == np.mean([apfds["dsa"][i] for i in sorted(apfds["dsa"])])
    # an approach without results, and one without CAM orders
    for cs in O.CASE_STUDIES:
        for ds in ("nominal", "ood"):
            assert df.loc[("surprise", "pc-mmdsa"), (cs, ds)] == "n.a."
            assert df.loc[("neuron coverage", "TKNC_3-cam"), (cs, ds)] == "n.a."
        assert df.loc[("surprise", "pc-mmdsa"), (cs, "time")] != df.loc[("surprise", "pc-mmdsa"), (cs, "time")]  # NaN
    assert df.loc[("uncertainty", "VR"), ("cifar10", "time")] == "n.a."
    assert df.loc[("uncertainty", "VR"), ("cifar10", "nominal")] == "n.a."
    # a time cell by hand: the model ids below 10, both datasets
    runs = [R.load_times(folder, "fmnist", ds, i, "KMNC_2") for ds in ("nominal", "ood") for i in O.MODEL_IDS if i < 10]
    setup, pred, quant, cam = (np.mean([t[k] for t in runs]) for k in range(4))
    assert df.loc[("neuron coverage", "KMNC_2"), ("fmnist", "time")] == f"{round(setup + 2 * (pred + quant))}s"
    assert df.loc[("neuron coverage", "KMNC_2-cam"), ("fmnist", "time")] == \
        f"{round(setup + 2 * (pred + quant + cam))}s"


def test_no_time_files_raise(folder, tmp_path):
    out = tmp_path / "out"
    shutil.copytree(os.path.join(folder, "priorities"), out / "priorities")
    with pytest.raises(ValueError, match="no time file"):
        R.apfd_table(str(out))
    os.makedirs(out / "times")
    with open(out / "times" / "mnist_nominal_10_dsa", "wb") as f:      # only model ids the table does not time
        pickle.dump([1.0, 1.0, 1.0, 1.0], f)
    with pytest.raises(ValueError, match="no time file"):
        R.write_apfd_table(str(out))
    assert not os.path.exists(out / "results")


def test_a_tip_without_time_files_in_one_case_study_gets_na_in_its_own_rows(folder, tmp_path):
    out = tmp_path / "out"
    shutil.copytree(folder, out)
    for f in os.listdir(out / "times"):
        if f.startswith("fmnist_") and (f.endswith("_VR") or f.endswith("_dsa")):
            os.remove(out / "times" / f)
    df = R.apfd_table(str(out))
    full = R.apfd_table(folder)
    assert df.loc[("uncertainty", "VR"), ("fmnist", "time")] == "n.a."
    assert df.loc[("surprise", "dsa"), ("fmnist", "time")] == "n.a."
    assert df.loc[("surprise", "dsa-cam"), ("fmnist", "time")] == "n.a."
    changed = [(row, col) for row in df.index for col in df.columns
               if str(df.loc[row, col]) != str(full.loc[row, col])]
    assert sorted(changed) == sorted([(("uncertainty", "VR"), ("fmnist", "time")),
                                      (("surprise", "dsa"), ("fmnist", "time")),
                                      (("surprise", "dsa-cam"), ("fmnist", "time"))])


def test_only_the_requested_case_studies(folder):
    df = R.apfd_table(folder, ["cifar10"])
    full = R.apfd_table(folder)
    assert list(df.columns) == [("cifar10", c) for c in ("nominal", "ood", "time")]
    assert df.equals(full[["cifar10"]])
