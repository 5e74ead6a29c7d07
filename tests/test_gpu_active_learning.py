"""The active-learning driver (core/active_learning.py) on the GPU with the real arms: every selection against the
reference's expression applied to `get_pred_and_uncertainty`, `CoverageWorker` and `SurpriseHandler` run on their own
on host copies of the observed splits, NumPy against CUDA-tensor inputs, and every accuracy against a NumPy
recomputation from the models' outputs."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NC_LAYERS, SA_LAYERS = [0, 2, 4], [4]
NUM_SELECTED, SHARE, MODEL_ID, SEED = 20, 0.5, 5, 2024


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


def _by_class(torch, model, per_class, rng, scale=1.0, pool=40_000):
    """(x, labels) as CUDA tensors: `per_class` inputs of each of the 3 classes, labelled with the model's clear top-1
    prediction."""
    x = torch.from_numpy((rng.normal(size=(pool, 1, 12, 12)) * scale).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x)
    top = z.topk(2, dim=1).values
    pred = z.argmax(dim=1).cpu().numpy()
    clear = ((top[:, 0] - top[:, 1]) > 1e-3).cpu().numpy()
    rows = [np.flatnonzero((pred == c) & clear)[:per_class] for c in range(3)]
    assert all(r.size == per_class for r in rows), "the toy model predicts a class too rarely"
    rows = np.concatenate(rows)
    return x[torch.from_numpy(rows).cuda()], torch.from_numpy(pred[rows].astype(np.int64)).cuda()


def _data(torch, model):
    rng = np.random.default_rng(0)
    train_x, train_y = _by_class(torch, model, 150, rng)
    nom_x, nom_y = _by_class(torch, model, 100, rng)
    ood_x, ood_y = _by_class(torch, model, 80, rng, scale=1.3)
    return {"train_x": train_x, "train_y": train_y, "nominal_test_x": nom_x, "nominal_test_labels": nom_y,
            "ood_test_x": ood_x, "ood_test_labels": ood_y}


def _run(torch, model, data, out_dir):
    """evaluate() with a spy on the global-RNG permutations and a deterministic training process whose models differ:
    a copy of the model whose last bias moves with the labels at the head of the data it received."""
    from simple_tip_b200.core import active_learning as AL

    draws, handed, models = [], [], []
    permutation = np.random.permutation

    def spy(n):
        perm = permutation(n)
        draws.append(perm.copy())
        return perm

    def training_process(x, y):
        handed.append((x.cpu().numpy(), y.cpu().numpy(), {x.device.type, y.device.type}))
        m = copy.deepcopy(model)
        with torch.no_grad():
            m[-2].bias += (y[:64].sum(dim=0).to(m[-2].bias.device) / 64 - 1 / 3) * 4.0
        models.append(m)
        return m
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(np.random, "permutation", spy)
        np.random.seed(SEED)
        out = AL.evaluate(MODEL_ID, "toy", model, nc_activation_layers=NC_LAYERS, sa_activation_layers=SA_LAYERS,
                          training_process=training_process, observed_share=SHARE, num_selected=NUM_SELECTED,
                          num_classes=3, output_folder=str(out_dir), **data)
    return out, draws, handed, models


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    torch = _torch()
    model = _toy_model(torch)
    data = _data(torch, model)
    host = {k: v.cpu().numpy() if isinstance(v, torch.Tensor) else v for k, v in data.items()}
    res = {}
    for name, d in (("cuda", data), ("numpy", host)):
        res[name] = _run(torch, model, d, tmp_path_factory.mktemp(name))
    return model, host, res


def _splits(host):
    from simple_tip_b200.core import active_learning as AL

    out = {}
    for name, x, y in (("nominal", host["nominal_test_x"], host["nominal_test_labels"]),
                       ("ood", host["ood_test_x"], host["ood_test_labels"])):
        obs, fut = AL.split_indices(len(x), SHARE, MODEL_ID)
        out[name, "observed"], out[name, "future"] = (x[obs], y[obs]), (x[fut], y[fut])
    return out


def test_selections_equal_the_arms_run_on_their_own(runs):
    from simple_tip_b200.core.activations import get_pred_and_uncertainty
    from simple_tip_b200.core.coverage_worker import CoverageWorker
    from simple_tip_b200.core.surprise_handler import SurpriseHandler

    model, host, res = runs
    (_, selections, _), _, _, _ = res["cuda"]
    obs = {name: xy[0] for (name, part), xy in _splits(host).items() if part == "observed"}
    k = NUM_SELECTED
    want = {}
    np.random.seed(SEED)                     # the arms in the driver's order, from the same global-RNG state
    for name, x in obs.items():
        _, unc, _ = get_pred_and_uncertainty(model, x)
        assert "VR" in unc
        for m, u in unc.items():
            want[m, name] = np.argsort(u)[-k:]
    worker = CoverageWorker(model, NC_LAYERS, host["train_x"])
    for name, x in obs.items():
        _, scores, orders = worker.evaluate_all(x)
        for m, s in scores.items():
            want[m, name] = np.argsort(s)[-k:]
        for m, o in orders.items():
            want[f"{m}-cam", name] = o[:k]
    for m, per_ds in SurpriseHandler(model, SA_LAYERS, host["train_x"]).evaluate_all(obs).items():
        for name, (s, order, _) in per_ds.items():
            want[m, name] = np.argsort(s)[-k:]
            want[f"{m}-cam", name] = order[:k]
    for name in obs:
        want["random", name] = list(range(k))
    assert set(selections) == set(want) and len(selections) == 80
    for key, sel in selections.items():
        np.testing.assert_array_equal(np.asarray(sel), np.asarray(want[key]), err_msg=str(key))


def test_numpy_and_cuda_inputs_agree(runs):
    _, host, res = runs
    (orig_c, sel_c, acc_c), draws_c, handed_c, _ = res["cuda"]
    (orig_n, sel_n, acc_n), draws_n, handed_n, _ = res["numpy"]
    assert list(sel_c) == list(sel_n)
    for key in sel_c:
        np.testing.assert_array_equal(np.asarray(sel_c[key]), np.asarray(sel_n[key]), err_msg=str(key))
    assert len(draws_c) == len(draws_n) == len(sel_c)
    n_train = host["train_x"].shape[0]
    for a, b in zip(draws_c, draws_n):
        assert a.shape == (n_train + NUM_SELECTED,)
        np.testing.assert_array_equal(a, b)
    for (xc, yc, dev_c), (xn, yn, dev_n) in zip(handed_c, handed_n):
        assert dev_c == {"cuda"} and dev_n == {"cpu"}
        np.testing.assert_array_equal(xc, xn)
        np.testing.assert_array_equal(yc, yn)
        assert yc.dtype == np.float32 and yc.shape == (n_train + NUM_SELECTED, 3)
    assert orig_c == orig_n and acc_c == acc_n


def test_handed_over_data_is_the_shuffled_merge(runs):
    _, host, res = runs
    (_, selections, _), draws, handed, _ = res["cuda"]
    splits = _splits(host)
    for ((_, name), idx), perm, (x, y, _) in zip(selections.items(), draws, handed):
        ox, oy = splits[name, "observed"]
        idx = np.asarray(idx)
        np.testing.assert_array_equal(x, np.concatenate((host["train_x"], ox[idx]))[perm])
        labels = np.concatenate((host["train_y"], oy[idx]))[perm]
        np.testing.assert_array_equal(y, np.eye(3, dtype=np.float32)[labels])


def test_accuracies_equal_a_numpy_recomputation(runs):
    torch = _torch()
    model, host, res = runs
    (orig, selections, accs), _, _, models = res["cuda"]
    splits = _splits(host)

    def host_acc(m):
        out = {}
        for key, (x, y) in splits.items():
            with torch.no_grad():
                p = np.concatenate([m(torch.from_numpy(x[i:i + 128]).cuda()).cpu().numpy()
                                    for i in range(0, len(x), 128)])
            out[key] = np.count_nonzero(np.argmax(p, axis=1) == y) / y.shape[0]
        return out
    assert orig == host_acc(model)
    assert list(accs) == list(selections) and len(models) == len(selections)
    for (key, acc), m in zip(accs.items(), models):
        assert acc == host_acc(m), key
    assert len({tuple(a.values()) for a in accs.values()}) > 1, "every retrained model scored the same"
