"""The prioritization driver (core/prioritization.py) on the GPU with the real arms: every result file against
`get_pred_and_uncertainty`, `CoverageWorker` and `SurpriseHandler` run on their own on host copies of the inputs,
CUDA-tensor against NumPy inputs, the time files, the returned APFDs against the folder's, Table 1 of two models,
and the caller's model left as it was."""
import os
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NC_LAYERS, SA_LAYERS = [0, 2, 4], [4]
MODEL_IDS, SEED, CASE_STUDY = (0, 1), 2024, "toy"
UNCERTAINTIES = ["softmax", "pcs", "softmax_entropy", "deep_gini", "VR"]


def _torch():
    import torch

    return torch


def _toy_model(torch):
    """A small conv net with a dropout layer (so VR is scored) whose last bias is shifted so that it predicts its 3
    classes about equally often on normal noise."""
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Conv2d(1, 4, 3), torch.nn.ReLU(), torch.nn.MaxPool2d(2), torch.nn.Flatten(),
                                torch.nn.Linear(4 * 5 * 5, 24), torch.nn.ReLU(), torch.nn.Dropout(0.3),
                                torch.nn.Linear(24, 3), torch.nn.Softmax(dim=1)).cuda().eval()
    x = torch.from_numpy(np.random.default_rng(99).normal(size=(20_000, 1, 12, 12)).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x).double().cpu().numpy()
    bias, step = np.zeros(3), z.std(axis=0).mean()
    for it in range(500):
        freq = np.bincount((z + bias).argmax(axis=1), minlength=3) / z.shape[0]
        bias -= step * 2.0 * (freq - 1 / 3) * 0.99 ** it
    with torch.no_grad():
        model[-2].bias += torch.from_numpy(bias).float().cuda()
    return model


def _by_class(torch, model, per_class, rng, scale=1.0, pool=40_000, wrong=0.2):
    """(x, labels) as CUDA tensors: `per_class` inputs of each of the 3 classes on which the model's top-1 is clear,
    labelled with that prediction, except for a share `wrong` of them, moved to another class."""
    x = torch.from_numpy((rng.normal(size=(pool, 1, 12, 12)) * scale).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x)
    top = z.topk(2, dim=1).values
    pred = z.argmax(dim=1).cpu().numpy()
    clear = ((top[:, 0] - top[:, 1]) > 1e-3).cpu().numpy()
    rows = [np.flatnonzero((pred == c) & clear)[:per_class] for c in range(3)]
    assert all(r.size == per_class for r in rows), "the toy model predicts a class too rarely"
    rows = np.concatenate(rows)
    labels = pred[rows].astype(np.int64)
    flip = rng.random(labels.size) < wrong
    labels[flip] = (labels[flip] + rng.integers(1, 3, int(flip.sum()))) % 3
    return x[torch.from_numpy(rows).cuda()], torch.from_numpy(labels).cuda()


def _data(torch, model):
    rng = np.random.default_rng(0)
    train_x, _ = _by_class(torch, model, 150, rng)
    nom_x, nom_y = _by_class(torch, model, 100, rng)
    ood_x, ood_y = _by_class(torch, model, 80, rng, scale=1.3)
    return {"training_dataset": train_x, "nominal_test_dataset": nom_x, "nominal_test_labels": nom_y,
            "ood_test_dataset": ood_x, "ood_test_labels": ood_y.reshape(-1, 1)}


def _state(model):
    return ({k: v.detach().cpu().clone() for k, v in model.state_dict().items()},
            [m.training for m in model.modules()])


def _npy_files(out):
    folder = os.path.join(out, "priorities")
    return {f: np.load(os.path.join(folder, f)) for f in sorted(os.listdir(folder))}


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    from simple_tip_b200.core import prioritization as P

    torch = _torch()
    model = _toy_model(torch)
    data = _data(torch, model)
    host = {k: v.cpu().numpy() for k, v in data.items()}
    before = _state(model)
    res = {}
    for name, d in (("cuda", data), ("numpy", host)):
        out = str(tmp_path_factory.mktemp(name))
        apfds = {}
        for model_id in MODEL_IDS:
            np.random.seed(SEED + model_id)            # sklearn's unseeded fits draw from the global RNG
            apfds[model_id] = P.evaluate(model_id, CASE_STUDY, model, nc_activation_layers=NC_LAYERS,
                                         sa_activation_layers=SA_LAYERS, output_folder=out, **d)
        res[name] = (out, apfds)
    return model, host, before, res


def _expected_files(model, host, model_id):
    """{file name: array} of one model: the arms run on their own on host copies, in the driver's order, from the
    global-RNG state the driver started from."""
    from simple_tip_b200.core.activations import get_pred_and_uncertainty
    from simple_tip_b200.core.coverage_worker import CoverageWorker
    from simple_tip_b200.core.surprise_handler import SurpriseHandler

    sets = {"nominal": (host["nominal_test_dataset"], host["nominal_test_labels"]),
            "ood": (host["ood_test_dataset"], host["ood_test_labels"])}
    want = {}
    np.random.seed(SEED + model_id)
    for ds, (x, y) in sets.items():
        pred, unc, _ = get_pred_and_uncertainty(model, x)
        assert list(unc) == UNCERTAINTIES
        want[f"{CASE_STUDY}_{ds}_{model_id}_is_misclassified.npy"] = pred != y.reshape(-1)
        for q, u in unc.items():
            want[f"{CASE_STUDY}_{ds}_{model_id}_uncertainty_{q}.npy"] = u
    worker = CoverageWorker(model, NC_LAYERS, host["training_dataset"])
    for ds, (x, _) in sets.items():
        _, scores, orders = worker.evaluate_all(x)
        for m in scores:
            want[f"{CASE_STUDY}_{ds}_{model_id}_{m}_scores.npy"] = scores[m]
            want[f"{CASE_STUDY}_{ds}_{model_id}_{m}_cam_order.npy"] = orders[m]
    del worker
    res = SurpriseHandler(model, SA_LAYERS, host["training_dataset"]).evaluate_all({ds: x for ds, (x, _) in
                                                                                     sets.items()})
    for m, per_ds in res.items():
        for ds, (s, order, _) in per_ds.items():
            want[f"{CASE_STUDY}_{ds}_{model_id}_{m}_scores.npy"] = s
            want[f"{CASE_STUDY}_{ds}_{model_id}_{m}_cam_order.npy"] = order
    return want


def test_files_equal_the_arms_run_on_their_own(runs):
    model, host, _, res = runs
    out, _ = res["cuda"]
    got = _npy_files(out)
    want = {}
    for model_id in MODEL_IDS:
        want.update(_expected_files(model, host, model_id))
    assert sorted(got) == sorted(want)
    assert len(want) == 2 * len(MODEL_IDS) * (1 + 5 + 2 * 12 + 2 * 5)
    for f, w in want.items():
        w = np.asarray(w)
        assert got[f].dtype == w.dtype, f
        assert np.array_equal(got[f], w), f
    for model_id in MODEL_IDS:
        for ds in ("nominal", "ood"):
            mask = got[f"{CASE_STUDY}_{ds}_{model_id}_is_misclassified.npy"]
            assert mask.dtype == bool and 0 < mask.sum() < mask.size


def test_cuda_and_numpy_inputs_write_the_same_files(runs):
    _, _, _, res = runs
    cuda, numpy = _npy_files(res["cuda"][0]), _npy_files(res["numpy"][0])
    assert sorted(cuda) == sorted(numpy)
    for f in cuda:
        assert cuda[f].dtype == numpy[f].dtype and np.array_equal(cuda[f], numpy[f]), f
    assert sorted(os.listdir(os.path.join(res["cuda"][0], "times"))) == \
        sorted(os.listdir(os.path.join(res["numpy"][0], "times")))


def test_time_files(runs):
    from simple_tip_b200.core.surprise_handler import SurpriseHandler

    _, _, _, res = runs
    for out, _ in res.values():
        folder = os.path.join(out, "times")
        metrics = UNCERTAINTIES + ["NBC_0", "NBC_0.5", "NBC_1", "SNAC_0", "SNAC_0.5", "SNAC_1", "NAC_0", "NAC_0.75",
                                   "TKNC_1", "TKNC_2", "TKNC_3", "KMNC_2"] + list(SurpriseHandler.TESTED_SA)
        assert sorted(os.listdir(folder)) == sorted(f"{CASE_STUDY}_{ds}_{i}_{m}" for ds in ("nominal", "ood")
                                                    for i in MODEL_IDS for m in metrics)
        for f in os.listdir(folder):
            with open(os.path.join(folder, f), "rb") as fh:
                t = pickle.load(fh)
            assert isinstance(t, list) and len(t) == 4, f
            assert all(isinstance(v, (int, float)) and v >= 0 for v in t), (f, t)
            if f.split("_", 3)[3] in UNCERTAINTIES:
                assert t[0] == 0 and t[3] == 0, (f, t)


def test_returned_apfds_equal_the_folders_and_the_table(runs):
    from simple_tip_b200.core import results as R

    _, _, _, res = runs
    for out, apfds in res.values():
        for ds in ("nominal", "ood"):
            loaded = R.load_apfd_values(out, CASE_STUDY, ds)
            for model_id in MODEL_IDS:
                got = apfds[model_id][ds]
                assert list(got) == R.APPROACHES
                assert got == {a: loaded[a][model_id] for a in R.APPROACHES}
        table = R.apfd_table(out, [CASE_STUDY])
        for approach in R.APPROACHES:
            row = (R.category(approach), approach)
            for ds in ("nominal", "ood"):
                assert table.loc[row, (CASE_STUDY, ds)] == np.mean([apfds[i][ds][approach] for i in MODEL_IDS])
            assert str(table.loc[row, (CASE_STUDY, "time")]).endswith("s")


def test_the_model_is_left_as_it_was(runs):
    model, _, (params, modes), _ = runs
    now_params, now_modes = _state(model)
    assert now_modes == modes
    assert list(now_params) == list(params)
    for k, v in params.items():
        assert now_params[k].dtype == v.dtype and torch_equal_bits(now_params[k], v), k


def torch_equal_bits(a, b) -> bool:
    return a.shape == b.shape and bytes(a.contiguous().numpy().tobytes()) == bytes(b.contiguous().numpy().tobytes())
