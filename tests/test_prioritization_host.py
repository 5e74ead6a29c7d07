"""The prioritization driver (core/prioritization.py) on the host, with the three arms replaced by deterministic fakes
that tie their integer scores: the arms' call order and arguments, the release of the coverage worker before the
surprise handler, the exact set of result files, the returned APFDs against the folder's, the input checks, and the
folder as the reference's unmodified table script reads it."""
import os
import weakref

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from simple_tip_b200.core import prioritization as P            # noqa: E402
from simple_tip_b200.core import results as R                   # noqa: E402
from simple_tip_b200.core.apfd import apfd_from_order           # noqa: E402

UNCERTAINTIES = ["softmax", "pcs", "softmax_entropy", "deep_gini"]       # a dropout-free model: no VR
NC_METRICS = ["NBC_0", "NBC_0.5", "NBC_1", "SNAC_0", "SNAC_0.5", "SNAC_1", "NAC_0", "NAC_0.75", "TKNC_1", "TKNC_2",
              "TKNC_3", "KMNC_2"]
SAS = ["dsa", "pc-lsa", "pc-mdsa", "pc-mlsa", "pc-mmdsa"]
CALLS = []
LIVE = []


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _scores(x, j, levels):
    """tied integer scores from one input column"""
    return np.floor(_host(x).reshape(len(x), -1)[:, j % 4] * levels).astype(np.int64)


def _order(x, j):
    return np.argsort(-_host(x).reshape(len(x), -1)[:, (j + 1) % 4], kind="stable")


def _pred(x):
    return np.argmax(_host(x).reshape(len(x), -1)[:, :3], axis=1).astype(np.int64)


def fake_pred_and_uncertainty(model, x, **kw):
    CALLS.append(("fp", len(x), kw))
    unc = {m: _scores(x, j, 3).astype(np.float64) for j, m in enumerate(UNCERTAINTIES)}
    return _pred(x), unc, {m: [0, 0.25 * j, 0.5, 0] for j, m in enumerate(unc)}


class FakeWorker:
    def __init__(self, model, nc_layers, training_data, batch_size=128):
        CALLS.append(("nc_init", list(nc_layers), len(training_data), batch_size))
        LIVE.append(("worker", weakref.ref(self)))
        self.traces = torch.zeros(8)

    def evaluate_all(self, test_dataset, test_dataset_id=None):
        CALLS.append(("nc_eval", len(test_dataset), test_dataset_id))
        scores = {m: _scores(test_dataset, j, 4).astype(np.int32) for j, m in enumerate(NC_METRICS)}
        orders = {m: _order(test_dataset, j) for j, m in enumerate(NC_METRICS)}
        return {m: [1.0, 2.0, 0.5 * j, 0.25] for j, m in enumerate(NC_METRICS)}, scores, orders


class FakeHandler:
    def __init__(self, model, sa_layers, training_data, batch_size=128):
        assert all(r() is None for kind, r in LIVE if kind == "worker"), "the coverage worker is still alive"
        CALLS.append(("sa_init", list(sa_layers), len(training_data), batch_size))
        LIVE.append(("handler", weakref.ref(self)))
        self.traces = torch.zeros(8)

    def evaluate_all(self, datasets, dsa_badge_size=None):
        CALLS.append(("sa_eval", [(ds, len(x)) for ds, x in datasets.items()], dsa_badge_size))
        return {m: {ds: (_scores(x, j, 5) / 5.0, _order(x, j), [3.0, 1.0, 0.5 * j, 0.75])
                    for ds, x in datasets.items()} for j, m in enumerate(SAS)}


@pytest.fixture
def fakes(monkeypatch):
    from simple_tip_b200.core import activations, coverage_worker, surprise_handler

    CALLS.clear()
    LIVE.clear()
    monkeypatch.setattr(activations, "get_pred_and_uncertainty", fake_pred_and_uncertainty)
    monkeypatch.setattr(coverage_worker, "CoverageWorker", FakeWorker)
    monkeypatch.setattr(surprise_handler, "SurpriseHandler", FakeHandler)
    return CALLS


def _model():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Softmax(dim=1))


def _data(n_train=30, n_nom=60, n_ood=50, seed=0):
    rng = np.random.default_rng(seed)
    return {"training_dataset": rng.random((n_train, 4), dtype=np.float32),
            "nominal_test_dataset": rng.random((n_nom, 4), dtype=np.float32),
            "nominal_test_labels": rng.integers(0, 3, n_nom),
            "ood_test_dataset": rng.random((n_ood, 4), dtype=np.float32),
            "ood_test_labels": rng.integers(0, 3, (n_ood, 1))}


def _run(tmp_path, data, model_id=3, case_study="toy", **kw):
    return P.evaluate(model_id, case_study, _model(), nc_activation_layers=[0], sa_activation_layers=[1],
                      output_folder=str(tmp_path), batch_size=16, **data, **kw)


def test_arms_run_in_the_references_order_with_the_arguments(fakes, tmp_path):
    _run(tmp_path, _data(), dsa_badge_size=7)
    assert fakes == [("fp", 60, {}), ("fp", 50, {}),
                     ("nc_init", [0], 30, 16), ("nc_eval", 60, "nominal"), ("nc_eval", 50, "ood"),
                     ("sa_init", [1], 30, 16), ("sa_eval", [("nominal", 60), ("ood", 50)], 7)]
    assert all(r() is None for _, r in LIVE)


def test_result_files(fakes, tmp_path):
    data = _data()
    _run(tmp_path, data)
    prio = os.path.join(tmp_path, "priorities")
    want = {}
    for ds in ("nominal", "ood"):
        x, y = data[f"{ds}_test_dataset"], data[f"{ds}_test_labels"].reshape(-1)
        stem = f"toy_{ds}_3"
        pred, unc, _ = fake_pred_and_uncertainty(None, x)
        want[f"{stem}_is_misclassified.npy"] = pred != y
        for m, u in unc.items():
            want[f"{stem}_uncertainty_{m}.npy"] = u
        for j, m in enumerate(NC_METRICS):
            want[f"{stem}_{m}_scores.npy"] = _scores(x, j, 4).astype(np.int32)
            want[f"{stem}_{m}_cam_order.npy"] = _order(x, j)
        for j, m in enumerate(SAS):
            want[f"{stem}_{m}_scores.npy"] = _scores(x, j, 5) / 5.0
            want[f"{stem}_{m}_cam_order.npy"] = _order(x, j)
    assert sorted(os.listdir(prio)) == sorted(want)
    for f, w in want.items():
        got = np.load(os.path.join(prio, f))
        assert got.dtype == w.dtype and np.array_equal(got, w), f
    assert want["toy_ood_3_is_misclassified.npy"].shape == (50,)
    for ds in ("nominal", "ood"):
        assert 0 < want[f"toy_{ds}_3_is_misclassified.npy"].sum() < len(data[f"{ds}_test_dataset"])

    times = os.path.join(tmp_path, "times")
    metrics = UNCERTAINTIES + NC_METRICS + SAS
    assert sorted(os.listdir(times)) == sorted(f"toy_{ds}_3_{m}" for ds in ("nominal", "ood") for m in metrics)
    for ds in ("nominal", "ood"):
        for j, m in enumerate(UNCERTAINTIES):
            assert R.load_times(str(tmp_path), "toy", ds, 3, m) == [0, 0.25 * j, 0.5, 0]
        for j, m in enumerate(NC_METRICS):
            assert R.load_times(str(tmp_path), "toy", ds, 3, m) == [1.0, 2.0, 0.5 * j, 0.25]
        for j, m in enumerate(SAS):
            assert R.load_times(str(tmp_path), "toy", ds, 3, m) == [3.0, 1.0, 0.5 * j, 0.75]
    assert sorted(os.listdir(tmp_path)) == ["priorities", "times"]


def test_returned_apfds_equal_the_folders(fakes, tmp_path):
    data = _data()
    res = _run(tmp_path, data)
    assert list(res) == ["nominal", "ood"]
    approaches = [a for a in R.APPROACHES if a != "VR"]
    for ds in ("nominal", "ood"):
        assert list(res[ds]) == approaches and len(approaches) == 38
        loaded = R.load_apfd_values(str(tmp_path), "toy", ds)
        assert sorted(loaded) == sorted(approaches)
        assert res[ds] == {a: loaded[a][3] for a in approaches}
        # by hand: argsort(-scores) for plain scores, the stored order for -cam
        x, y = data[f"{ds}_test_dataset"], data[f"{ds}_test_labels"].reshape(-1)
        mask = _pred(x) != y
        _, unc, _ = fake_pred_and_uncertainty(None, x)
        for m, u in unc.items():
            assert res[ds][m] == apfd_from_order(mask, np.argsort(-u))
        for j, m in enumerate(NC_METRICS):
            assert res[ds][m] == apfd_from_order(mask, np.argsort(-_scores(x, j, 4).astype(np.int32)))
            assert res[ds][f"{m}-cam"] == apfd_from_order(mask, _order(x, j))
        for j, m in enumerate(SAS):
            assert res[ds][m] == apfd_from_order(mask, np.argsort(-(_scores(x, j, 5) / 5.0)))
            assert res[ds][f"{m}-cam"] == apfd_from_order(mask, _order(x, j))


def test_tensor_inputs_give_the_same_folder(fakes, tmp_path):
    data = _data()
    a = _run(tmp_path / "a", data)
    b = _run(tmp_path / "b", {k: torch.from_numpy(np.asarray(v)) for k, v in data.items()})
    assert a == b
    for f in os.listdir(tmp_path / "a" / "priorities"):
        x, y = np.load(tmp_path / "a" / "priorities" / f), np.load(tmp_path / "b" / "priorities" / f)
        assert x.dtype == y.dtype and np.array_equal(x, y), f


@pytest.mark.parametrize("key,labels", [("nominal_test_labels", np.zeros(59, np.int64)),
                                        ("ood_test_labels", np.zeros((50, 2), np.int64)),
                                        ("ood_test_labels", np.zeros((1, 50), np.int64)),
                                        ("nominal_test_labels", np.int64(0))])
def test_label_shape_mismatch_raises_before_any_arm(fakes, tmp_path, key, labels):
    data = _data()
    data[key] = labels
    with pytest.raises(ValueError, match=key):
        _run(tmp_path, data)
    assert not fakes and not os.path.exists(os.path.join(tmp_path, "priorities"))


def test_case_study_with_underscore_raises_before_any_arm(fakes, tmp_path):
    with pytest.raises(ValueError, match="my_cs"):
        _run(tmp_path, _data(), case_study="my_cs")
    assert not fakes and not os.listdir(tmp_path)


def test_the_model_is_left_as_it_was(fakes, tmp_path):
    model = _model()
    model[0].train()
    modes = [m.training for m in model.modules()]
    before = {k: v.clone() for k, v in model.state_dict().items()}
    P.evaluate(0, "toy", model, nc_activation_layers=[0], sa_activation_layers=[1], output_folder=str(tmp_path),
               **_data())
    assert [m.training for m in model.modules()] == modes
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k])


def test_the_references_table_script_reads_the_same_apfds(fakes, tmp_path):
    import warnings

    from oracle import ref_harness

    if not ref_harness.available():
        pytest.skip("the reference checkout is not available")
    from oracle.apfd_table_oracle import load_plotters

    res = {model_id: _run(tmp_path, _data(seed=model_id), model_id=model_id) for model_id in (0, 4)}
    ref = load_plotters(str(tmp_path))
    for ds in ("nominal", "ood"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")          # the reference warns about every approach missing on cifar10
            got = ref.eval_apfd_table.load_apfd_values("toy", ds)
        assert got == {a: {i: res[i][ds][a] for i in res} for a in res[0][ds]}
