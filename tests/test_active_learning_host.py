"""The active-learning driver (core/active_learning.py) on the host, with the three arms replaced by deterministic
fakes: the split, the selections and their order, the retraining hand-over and its global-RNG draws, the sanity
checks, the release of the arms' workers before retraining, and the result files as the reference's table script
reads them."""
import os
import pickle
import re
import weakref

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from simple_tip_b200.core import active_learning as AL          # noqa: E402

# eval_active_learning.py / handler_*.py names, in the order the reference's dicts hold them
UNCERTAINTIES = ["softmax", "pcs", "softmax_entropy", "deep_gini", "VR"]
NC_METRICS = ["NBC_0", "NBC_0.5", "NBC_1", "SNAC_0", "SNAC_0.5", "SNAC_1", "NAC_0", "NAC_0.75", "TKNC_1", "TKNC_2",
              "TKNC_3", "KMNC_2"]
SAS = ["dsa", "pc-lsa", "pc-mdsa", "pc-mlsa", "pc-mmdsa"]

# src/plotters/utils.py APPROACHES
APPROACHES = ["NAC_0.75-cam", "NAC_0.75", "NAC_0-cam", "NAC_0", "NBC_0.5-cam", "NBC_0.5", "NBC_0-cam", "NBC_0",
              "NBC_1-cam", "NBC_1", "SNAC_0.5-cam", "SNAC_0.5", "SNAC_0-cam", "SNAC_0", "SNAC_1-cam", "SNAC_1",
              "TKNC_1-cam", "TKNC_1", "TKNC_2-cam", "TKNC_2", "TKNC_3-cam", "TKNC_3", "KMNC_2-cam", "KMNC_2",
              "dsa-cam", "dsa", "pc-lsa-cam", "pc-lsa", "pc-mdsa-cam", "pc-mdsa", "pc-mlsa-cam", "pc-mlsa",
              "pc-mmdsa-cam", "pc-mmdsa", "deep_gini", "softmax", "pcs", "softmax_entropy", "VR"]


def reference_keys():
    """The selection keys in the insertion order of eval_active_learning.py:69-87."""
    keys = []
    for ds in ("nominal", "ood"):                                   # _get_fp_selection
        keys += [(m, ds) for m in UNCERTAINTIES]
    for ds in ("nominal", "ood"):                                   # _get_nc_selection
        keys += [(m, ds) for m in NC_METRICS] + [(f"{m}-cam", ds) for m in NC_METRICS]
    for m in SAS:                                                   # _get_sa_selection
        for ds in ("nominal", "ood"):
            keys += [(m, ds), (f"{m}-cam", ds)]
    return keys + [("random", "nominal"), ("random", "ood")]       # _get_random_section


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _scores(x, j, levels):
    """tied integer scores from one input column"""
    return np.floor(_host(x).reshape(len(x), -1)[:, j % 4] * levels).astype(np.int64)


def _order(x, j):
    return np.argsort(-_host(x).reshape(len(x), -1)[:, (j + 1) % 4], kind="stable")


LIVE = []


def fake_pred_and_uncertainty(model, x, **kw):
    unc = {m: _scores(x, j, 3).astype(np.float64) for j, m in enumerate(UNCERTAINTIES)}
    return np.zeros(len(x), np.int64), unc, {m: [0, 0, 0, 0] for m in unc}


class FakeWorker:
    def __init__(self, model, nc_layers, training_data, batch_size=128):
        LIVE.append(weakref.ref(self))
        self.traces = torch.zeros(8)

    def evaluate_all(self, test_dataset, test_dataset_id=None):
        scores = {m: _scores(test_dataset, j, 4).astype(np.int32) for j, m in enumerate(NC_METRICS)}
        orders = {m: _order(test_dataset, j) for j, m in enumerate(NC_METRICS)}
        return {m: [0, 0, 0, 0] for m in NC_METRICS}, scores, orders


class FakeHandler:
    def __init__(self, model, sa_layers, training_data, batch_size=128):
        LIVE.append(weakref.ref(self))
        self.traces = torch.zeros(8)

    def evaluate_all(self, datasets, dsa_badge_size=None):
        return {m: {ds: (_scores(x, j, 5) / 5.0, _order(x, j), [0, 0, 0, 0]) for ds, x in datasets.items()}
                for j, m in enumerate(SAS)}


@pytest.fixture
def fakes(monkeypatch):
    from simple_tip_b200.core import activations, coverage_worker, surprise_handler

    LIVE.clear()
    monkeypatch.setattr(activations, "get_pred_and_uncertainty", fake_pred_and_uncertainty)
    monkeypatch.setattr(coverage_worker, "CoverageWorker", FakeWorker)
    monkeypatch.setattr(surprise_handler, "SurpriseHandler", FakeHandler)
    draws = []
    permutation = np.random.permutation

    def spy(n):
        perm = permutation(n)
        draws.append(perm.copy())
        return perm
    monkeypatch.setattr(np.random, "permutation", spy)
    return draws


def _model():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Softmax(dim=1))


def _data(n_train=30, n_nom=60, n_ood=50, seed=0):
    rng = np.random.default_rng(seed)
    return {"train_x": rng.random((n_train, 4), dtype=np.float32), "train_y": rng.integers(0, 3, (n_train, 1)),
            "nominal_test_x": rng.random((n_nom, 4), dtype=np.float32), "nominal_test_labels": rng.integers(0, 3, n_nom),
            "ood_test_x": rng.random((n_ood, 4), dtype=np.float32), "ood_test_labels": rng.integers(0, 3, n_ood)}


def _run(tmp_path, data, num_selected=8, num_classes=3, training_process=None, model_id=3):
    calls = []

    def train(x, y):
        assert all(r() is None for r in LIVE), "an arm's worker is still alive at the first retraining"
        calls.append((x, y))
        m = _model()
        with torch.no_grad():
            m[0].bias += torch.tensor([0.1 * len(calls), 0.0, -0.1 * len(calls)])
        return m
    res = AL.evaluate(model_id, "toy", _model(), nc_activation_layers=[0], sa_activation_layers=[0],
                      training_process=training_process or train, observed_share=0.4, num_selected=num_selected,
                      num_classes=num_classes, output_folder=str(tmp_path), batch_size=16, **data)
    return res, calls


@pytest.mark.parametrize("n,share,model_id", [(10, 0.5, 0), (101, 0.5, 3), (257, 0.3, 17), (1000, 0.25, 99),
                                              (37, 0.9, 1)])
def test_split_equals_train_test_split_on_the_arrays(n, share, model_id):
    from sklearn.model_selection import train_test_split

    rng = np.random.default_rng(n)
    x, y = rng.random((n, 3)), rng.integers(0, 10, n)
    xo, yo = rng.random((n + 1, 2)), rng.integers(0, 10, n + 1)
    ds = AL._shuffle_and_split_datasets(model_id, x, y, xo, yo, observed_share=share)
    assert list(ds) == [("nominal", "observed"), ("nominal", "future"), ("ood", "observed"), ("ood", "future")]
    for name, (a, b) in (("nominal", (x, y)), ("ood", (xo, yo))):
        fut_x, obs_x, fut_y, obs_y = train_test_split(a, b, test_size=share, random_state=model_id)
        for got, want in zip(ds[name, "observed"] + ds[name, "future"], (obs_x, obs_y, fut_x, fut_y)):
            np.testing.assert_array_equal(got, want)
    # tensors are split on their own device with the same rows
    ts = AL._shuffle_and_split_datasets(model_id, torch.from_numpy(x), y, xo, torch.from_numpy(yo), share)
    for k in ds:
        for got, want in zip(ts[k], ds[k]):
            np.testing.assert_array_equal(_host(got), want)


@pytest.mark.parametrize("num_classes", [3, None])
def test_selections_retraining_and_accuracies(fakes, tmp_path, num_classes):
    data = _data()
    np.random.seed(123)
    (orig, sel, acc), calls = _run(tmp_path, data, num_classes=num_classes)
    assert list(sel) == reference_keys()

    ds = AL._shuffle_and_split_datasets(3, data["nominal_test_x"], data["nominal_test_labels"], data["ood_test_x"],
                                        data["ood_test_labels"], 0.4)
    obs = {"nominal": ds["nominal", "observed"], "ood": ds["ood", "observed"]}
    want = {}
    for name, (x, _) in obs.items():
        _, unc, _ = fake_pred_and_uncertainty(None, x)
        for m, u in unc.items():
            want[m, name] = np.argsort(u)[-8:]
        _, scores, orders = FakeWorker(None, [0], None).evaluate_all(x)
        for m in NC_METRICS:
            want[m, name] = np.argsort(scores[m])[-8:]
            want[f"{m}-cam", name] = orders[m][:8]
    for m, per_ds in FakeHandler(None, [0], None).evaluate_all({k: v[0] for k, v in obs.items()}).items():
        for name, (s, order, _) in per_ds.items():
            want[m, name] = np.argsort(s)[-8:]
            want[f"{m}-cam", name] = order[:8]
    for name in obs:
        want["random", name] = list(range(8))
    for k in sel:
        np.testing.assert_array_equal(np.asarray(sel[k]), np.asarray(want[k]), err_msg=str(k))

    # one global-RNG permutation per selection, in order, of the merged set's length; the hand-over is that merge
    assert len(fakes) == len(sel) == len(calls)
    np.random.seed(123)
    n_train = data["train_x"].shape[0]
    for (key, idx), perm, (x, y) in zip(sel.items(), fakes, calls):
        assert perm.shape == (n_train + 8,)
        np.testing.assert_array_equal(perm, np.random.permutation(n_train + 8))
        ox, oy = obs[key[1]]
        wx = np.concatenate((data["train_x"], ox[np.asarray(idx)]))[perm]
        wy = np.concatenate((data["train_y"].flatten(), oy[np.asarray(idx)].flatten()))[perm]
        assert isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor)
        np.testing.assert_array_equal(x.numpy(), wx)
        if num_classes is None:
            assert y.dtype == torch.int64
            np.testing.assert_array_equal(y.numpy(), wy)
        else:
            assert y.dtype == torch.float32 and y.shape == (n_train + 8, 3)
            np.testing.assert_array_equal(y.numpy(), np.eye(3, dtype=np.float32)[wy])

    # accuracies: argmax of the outputs against the labels, exactly, on all four splits
    def host_acc(model):
        out = {}
        for k, (x, y) in ds.items():
            with torch.no_grad():          # the driver's batches of 16
                p = np.concatenate([model(torch.from_numpy(x[i:i + 16])).numpy() for i in range(0, len(x), 16)])
            out[k] = np.count_nonzero(np.argmax(p, axis=1) == y) / y.shape[0]
        return out
    assert orig == host_acc(_model())
    for i, (k, res) in enumerate(acc.items()):
        m = _model()
        with torch.no_grad():
            m[0].bias += torch.tensor([0.1 * (i + 1), 0.0, -0.1 * (i + 1)])
        assert list(res) == list(ds) and res == host_acc(m), k
        assert all(type(v) is float for v in res.values())


def test_too_small_observed_split_raises_before_retraining(fakes, tmp_path):
    called = []
    with pytest.raises(AssertionError, match=re.escape(
            "The number of selected indexes for softmax, nominal is not correct.Should be 30, but was 24")):
        _run(tmp_path, _data(), num_selected=30, training_process=lambda x, y: called.append(1))
    assert not called and not fakes
    assert not os.path.exists(os.path.join(tmp_path, "active_learning"))


def test_result_files_as_the_table_script_reads_them(fakes, tmp_path):
    (orig, sel, acc), _ = _run(tmp_path, _data(), model_id=7)
    folder = os.path.join(tmp_path, "active_learning")
    files = sorted(os.listdir(folder))
    assert files == sorted([f"toy_7_{m}_{d}.pickle" for m, d in sel] + ["toy_7_original_na.pickle"])

    def load(f):
        with open(os.path.join(folder, f), "rb") as fh:
            return pickle.load(fh)
    assert load("toy_7_original_na.pickle") == orig
    for (m, d), res in acc.items():
        got = load(f"toy_7_{m}_{d}.pickle")
        assert got == res and list(got) == [("nominal", "observed"), ("nominal", "future"), ("ood", "observed"),
                                            ("ood", "future")]

    # eval_active_learning_table.py:26-59 (load_arrays_active_learning, by_id=True) over the folder
    def by_regex(pattern):
        regex = re.compile(pattern)
        return {int(f.split("_")[1]): load(f) for f in os.listdir(folder) if regex.match(f, pos=0)}
    for ds_name in ("nominal", "ood"):
        for approach in APPROACHES + ["random"]:
            found = by_regex(f"toy_\\d*_{approach}_{ds_name}\\.")
            assert found == {7: acc[approach, ds_name]}, (approach, ds_name)
    assert by_regex("toy_\\d*_original_na\\.") == {7: orig}
