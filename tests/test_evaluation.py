"""The study's evaluation phase without TensorFlow (core/evaluation.py): Table 2 and the Wilcoxon / A12 statistics
against the reference's src/plotters scripts on a seeded synthetic result folder (oracle/evaluation_oracle.py) — the
CSVs against golden copies of what the reference's `run()` wrote, the DataFrames and grids against the reference's
where its checkout exists — and the kept quirks, the p-value against a restatement of scipy 1.4.1's code path and
against scipy's own asymptotic test, A12 by hand and the missing-data cells."""
import os
import pickle
import shutil
import warnings

import numpy as np
import pytest

pytest.importorskip("pandas")

from oracle import apfd_table_oracle          # noqa: E402
from oracle import evaluation_oracle as O     # noqa: E402
from oracle import ref_harness                # noqa: E402
from simple_tip_b200.core import evaluation as E  # noqa: E402
from simple_tip_b200.core import results as R     # noqa: E402

STATISTICS = {"test_prio_statistics": ("apfd_correlation_p.csv", "apfd_correlation_eff.csv"),
              "active_learning_statistics": ("active_correlation_p.csv", "active_correlation_eff.csv")}


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    return O.write(str(tmp_path_factory.mktemp("results") / "out"))


@pytest.fixture
def copy(folder, tmp_path):
    out = str(tmp_path / "out")
    shutil.copytree(folder, out)
    return out


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _statistics_bytes(out, eval_type):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return [_read(p) for p in E.evaluate_results(out, eval_type)]


def test_csvs_equal_the_references_byte_for_byte(copy):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        written = {t: E.evaluate_results(copy, t) for t in E.EVAL_TYPES}
    results = os.path.join(copy, "results")
    assert written == {"test_prio": [os.path.join(results, "apfds.csv")],
                       "active_learning": [os.path.join(results, "active.csv")],
                       **{t: [os.path.join(results, n) for n in names] for t, names in STATISTICS.items()}}
    assert _read(os.path.join(results, "apfds.csv")) == _read(apfd_table_oracle.GOLDEN_CSV)
    for name, golden in O.GOLDEN.items():
        assert _read(os.path.join(results, name)) == _read(golden), name
    assert sorted(os.listdir(results)) == sorted(["apfds.csv"] + list(O.GOLDEN))


def test_dataframes_and_grids_equal_the_references(folder):
    if not ref_harness.available():
        pytest.skip("the reference checkout is not available")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mine = E.active_learning_table(folder)
    ref = O.reference_table(folder)
    assert mine.index.equals(ref.index) and mine.columns.equals(ref.columns)
    assert mine.equals(ref)
    assert O.reference_run(folder, "active_learning") == ({"active.csv": _read(O.GOLDEN["active.csv"])}, None)
    for eval_type, statistics in (("test_prio_statistics", E.apfd_statistics),
                                  ("active_learning_statistics", E.active_learning_statistics)):
        files, ref_grids = O.reference_run(folder, eval_type)
        assert files == {name: _read(O.GOLDEN[name]) for name in STATISTICS[eval_type]}
        grids, _ = statistics(folder)
        assert sorted(grids) == sorted(ref_grids)
        for k in grids:
            assert grids[k].dtype.kind == ref_grids[k].dtype.kind
            np.testing.assert_array_equal(grids[k], ref_grids[k], err_msg=f"{eval_type} {k}")


def _runs(folder, case_study, approach, ds):
    """The top-level result pickles of an approach, by model id."""
    al = os.path.join(folder, "active_learning")
    out = {}
    for f in os.listdir(al):
        if not os.path.isfile(os.path.join(al, f)):
            continue
        cs, model_id, rest = f.split("_", 2)
        if cs == case_study and rest in (f"{approach}_{ds}.pickle", f"{approach.replace('.', 'x')}_{ds}.pickle"):
            with open(os.path.join(al, f), "rb") as fh:
                out[int(model_id)] = pickle.load(fh)
    return out


def test_table_cells(folder):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        df = E.active_learning_table(folder)
    # one warning per missing approach, none for VR on cifar10
    assert [str(w.message) for w in caught] == ["missing results"] * len(O.MISSING)
    assert list(df.index) == [(R.category(a), a) for a in ["original", "random"] + R.APPROACHES]
    assert df.index.get_level_values(0)[0] == "baseline"
    key = ("ood", "future")
    for approach in ("original", "random"):
        ds = "na" if approach == "original" else "nominal"
        runs = _runs(folder, "imdb", approach, ds)
        assert len(runs) == len(O.MODEL_IDS)
        mean = np.mean([r[key] for r in runs.values()])
        assert df.at[("baseline", approach), ("imdb", "nominal", "ood:future")] == f"{mean:.2%}"
    # a TIP's cell is its mean less random's; NAC_0.75's runs include the file named NAC_0x75
    nac = _runs(folder, "fmnist", "NAC_0.75", "ood")
    assert len(nac) == len(O.MODEL_IDS)
    rnd = _runs(folder, "fmnist", "random", "ood")
    gain = np.mean([r[key] for r in nac.values()]) - np.mean([r[key] for r in rnd.values()])
    assert df.at[("neuron coverage", "NAC_0.75"), ("fmnist", "ood", "ood:future")] == f"{gain:.2%}"
    # the subfolder's copy is read from the top-level folder: that file counts twice
    dsa = _runs(folder, "mnist", "dsa", "nominal")
    values = [r[key] for r in dsa.values()] + [dsa[2][key]]
    rnd = [r[key] for r in _runs(folder, "mnist", "random", "nominal").values()]
    assert df.at[("surprise", "dsa"), ("mnist", "nominal", "ood:future")] == f"{np.mean(values) - np.mean(rnd):.2%}"
    # missing approaches
    for cs, ds, approach in sorted(O.MISSING) + [("cifar10", "nominal", "VR"), ("cifar10", "ood", "VR")]:
        row = (R.category(approach), approach)
        assert [df.at[row, (cs, ds, s)] for s in ("nominal:observed", "nominal:future", "ood:observed",
                                                  "ood:future")] == ["n.a."] * 4
    assert df.notna().all().all()


def test_cells_no_run_names_stay_empty(copy):
    al = os.path.join(copy, "active_learning")
    for f in os.listdir(al):
        if f.startswith("imdb_") and f.endswith("_dsa_ood.pickle"):
            with open(os.path.join(al, f), "rb") as fh:
                res = pickle.load(fh)
            del res[("nominal", "observed")]
            with open(os.path.join(al, f), "wb") as fh:
                pickle.dump(res, fh)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        df = E.active_learning_table(copy)
        E.write_active_learning_table(copy)
    row = ("surprise", "dsa")
    assert df.loc[row, ("imdb", "ood", "nominal:observed")] != df.loc[row, ("imdb", "ood", "nominal:observed")]
    assert df.isna().sum().sum() == 1
    line = [ln for ln in _read(os.path.join(copy, "results", "active.csv")).decode().splitlines()
            if ln.startswith("surprise,dsa,")][0]
    assert line.split(",")[2 + 3 * 8 + 4] == ""


def test_random_is_required(copy):
    al = os.path.join(copy, "active_learning")
    for f in os.listdir(al):
        if f.startswith("cifar10_") and f.endswith("_random_ood.pickle"):
            os.remove(os.path.join(al, f))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        E.active_learning_table(copy, ["mnist"])
        with pytest.raises(AssertionError):
            E.active_learning_table(copy)


def _rewrite_npy(path, f):
    np.save(path, f(np.load(path)))


def test_apfd_statistics_compare_ood_values_only(copy):
    before = _statistics_bytes(copy, "test_prio_statistics")
    priorities = os.path.join(copy, "priorities")
    old = R.load_apfd_values(copy, "mnist", "nominal")["dsa"][3]
    _rewrite_npy(os.path.join(priorities, "mnist_nominal_3_dsa_scores.npy"), lambda s: -s)
    assert R.load_apfd_values(copy, "mnist", "nominal")["dsa"][3] != old
    assert _statistics_bytes(copy, "test_prio_statistics") == before
    _rewrite_npy(os.path.join(priorities, "mnist_ood_3_dsa_scores.npy"), lambda s: -s)
    after = _statistics_bytes(copy, "test_prio_statistics")
    assert after[0] != before[0] and after[1] != before[1]


def test_active_learning_statistics_compare_ood_values_only(copy):
    before = _statistics_bytes(copy, "active_learning_statistics")
    for ds, change in (("nominal", False), ("ood", True)):
        path = os.path.join(copy, "active_learning", f"mnist_9_dsa_{ds}.pickle")
        with open(path, "rb") as f:
            res = pickle.load(f)
        res[(ds, "future")] += 0.31
        with open(path, "wb") as f:
            pickle.dump(res, f)
        after = _statistics_bytes(copy, "active_learning_statistics")
        assert (after != before) == change, ds


def test_statistics_missing_data_cells(folder):
    grids, missing = E.active_learning_statistics(folder)
    idx = {a: i for i, a in enumerate(R.APPROACHES)}
    n = len(R.APPROACHES)
    stat_ids = [i for i in O.MODEL_IDS if i < 100]
    # no shared sample: pc-mmdsa-cam and pc-mmdsa ran on different models
    i, j = idx["pc-mmdsa-cam"], idx["pc-mmdsa"]
    assert grids["num_samples"][i, j] == 0 and np.isnan(grids["p"][i, j]) and np.isnan(grids["e"][i, j])
    # identical samples: SNAC_1 repeats SNAC_0
    i, j = idx["SNAC_0"], idx["SNAC_1"]
    assert grids["num_samples"][i, j] == len(O.CASE_STUDIES) * len(stat_ids)
    assert np.isnan(grids["p"][i, j]) and np.isnan(grids["e"][i, j])
    # the fill of the diagonal and the lower triangle
    lower = np.tril(np.ones((n, n), dtype=bool))
    assert (grids["p"][lower] == E.P_FILL).all() and (grids["e"][lower] == E.E_FILL).all()
    assert (grids["num_samples"][lower] == E.NUM_SAMPLES_FILL).all()
    upper = ~lower & ~np.isnan(grids["p"])
    assert ((grids["p"][upper] > 0) & (grids["p"][upper] <= 1)).all()
    assert ((grids["e"][upper] >= 0) & (grids["e"][upper] <= 1)).all()
    # the runs some approach lacks: all, as pc-mmdsa-cam and pc-mmdsa each have one model
    assert missing == {(cs, ds): set(range(100)) for cs in O.CASE_STUDIES for ds in ("nominal", "ood")}
    p, e = E.statistics_frames(grids)
    names = list(p.index)
    assert names[:2] == ["NAC-0.75-CAM", "NAC-0.75"] and names[-5:] == ["DeepGini", "Vanilla SM", "PCS", "Entropy",
                                                                        "MC-Dropout"]
    assert p.iloc[1, 0] == "" and e.iloc[1, 0] == E.E_FILL


def test_evaluate_results_warns_missing_runs_and_rejects_unknown_types(copy):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        E.evaluate_results(copy, "test_prio_statistics")
    ids = sorted(set(range(100)) - {i for i in apfd_table_oracle.MODEL_IDS if i < 100})
    assert [str(w.message) for w in caught] == [f"Missing values {cs} - {ds}: {ids}" for cs in O.CASE_STUDIES
                                                for ds in ("nominal", "ood")]
    with pytest.raises(ValueError, match="unknown evaluation type"):
        E.evaluate_results(copy, "evaluation")


def _cases():
    rng = np.random.default_rng(7)
    for n in (2, 9, 10, 24, 25, 26, 50, 51, 120, 800):
        x = rng.integers(0, 12, n) / 10                        # ties among |d| and zero differences
        y = rng.integers(0, 12, n) / 10
        if np.any(x != y):
            yield x, y
        yield rng.random(n), rng.random(n)
    yield np.arange(60.0), np.arange(60.0) - 1                  # one tie group of all differences
    yield np.r_[np.zeros(30), np.ones(5)], np.zeros(35)        # mostly zeros


def test_wilcoxon_p_matches_scipy_141s_normal_approximation():
    cases = list(_cases())
    assert len(cases) > 20
    for x, y in cases:
        want = O.scipy141_wilcoxon_p(x, y)
        got = E.wilcoxon_p(list(x), list(y))
        assert got == pytest.approx(want, rel=1e-12, abs=0), (len(x), got, want)
    with pytest.raises(ValueError):
        E.wilcoxon_p([0.5, 0.25], [0.5, 0.25])


def test_wilcoxon_p_matches_scipys_asymptotic_test_without_ties():
    from scipy import stats

    rng = np.random.default_rng(11)
    for n in (51, 90, 400, 800):
        x, y = rng.random(n), rng.random(n) + 0.05 * rng.standard_normal()
        assert len(np.unique(np.abs(x - y))) == n and np.all(x != y)
        want = stats.wilcoxon(x, y, alternative="two-sided", method="asymptotic").pvalue
        assert E.wilcoxon_p(x, y) == pytest.approx(want, rel=1e-12, abs=0), n


def test_a12_by_hand():
    assert E.paired_a12([2, 3, 4, 5], [1, 2, 3, 4]) == 1.0          # all greater
    assert E.paired_a12([1, 2, 3, 4], [2, 3, 4, 5]) == 1.0          # all smaller
    assert E.paired_a12([1, 2, 3, 4], [1, 2, 3, 4]) == 0.0          # all equal
    assert E.paired_a12([2, 3, 3, 4], [1, 2, 4, 5]) == 0.0          # half greater, half smaller
    assert E.paired_a12([2, 3, 3, 4], [1, 2, 3, 4]) == 0.5          # half greater, half equal: 2 * |0.75 - 0.5|
    assert E.paired_a12([1, 1, 1], [0, 0, 5]) == pytest.approx(1 / 3)


def test_wilcoxon_a12_grid():
    m = {"a": {"s1": 0.1, "s2": 0.2, "s3": 0.3}, "b": {"s2": 0.25, "s3": 0.1, "s4": 9.0},
         "c": {"s1": 0.1, "s2": 0.2}, "d": {"s4": 1.0}, "ignored": {"s1": 5.0}}
    g = E.wilcoxon_a12(m, ["a", "b", "c", "d"])
    assert g["num_samples"][0, 1] == 2 and g["num_samples"][0, 2] == 2 and g["num_samples"][0, 3] == 0
    assert g["p"][0, 1] == O.scipy141_wilcoxon_p([0.2, 0.3], [0.25, 0.1])
    assert g["e"][0, 1] == 0.0                                     # one greater, one smaller
    assert np.isnan(g["p"][0, 2]) and np.isnan(g["e"][0, 2])        # equal on their shared samples
    assert np.isnan(g["p"][0, 3]) and np.isnan(g["e"][0, 3])        # no shared sample
    assert g["e"][1, 3] == 1.0 and g["num_samples"][1, 3] == 1
    assert g["p"][1, 0] == E.P_FILL and g["e"][2, 2] == E.E_FILL and g["num_samples"][3, 0] == E.NUM_SAMPLES_FILL
