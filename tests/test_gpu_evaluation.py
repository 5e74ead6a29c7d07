"""The evaluation phase (core/evaluation.py) on result folders the GPU experiments wrote: `active_learning.evaluate`
and `prioritization.evaluate` for two models of a small CNN, with a few-step training process, into one folder, then
`evaluate_results` for all four evaluation types.  Table 2's cells against the accuracies the calls returned, the
statistics' effect sizes against A12 of the returned APFDs and accuracies (the OOD values only), and every file read
back."""
import copy
import os
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NC_LAYERS, SA_LAYERS = [0, 2, 4], [4]
MODEL_IDS, SEED, CASE_STUDY = (0, 1), 2024, "toy"
NUM_SELECTED, SHARE = 20, 0.5
SPLITS = ("nominal", "ood")


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


def _training_process(torch, model):
    """Three SGD steps of a copy of the model on the cross-entropy of its softmax output."""
    def train(x, y):
        m = copy.deepcopy(model).train()
        opt = torch.optim.SGD(m.parameters(), lr=0.5)
        for start in range(0, 3 * 128, 128):
            opt.zero_grad()
            loss = -(y[start:start + 128] * torch.log(m(x[start:start + 128]) + 1e-9)).sum(dim=1).mean()
            loss.backward()
            opt.step()
        return m.eval()
    return train


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    from simple_tip_b200.core import active_learning as AL
    from simple_tip_b200.core import evaluation as E
    from simple_tip_b200.core import prioritization as P

    torch = _torch()
    model = _toy_model(torch)
    rng = np.random.default_rng(0)
    train_x, train_y = _by_class(torch, model, 150, rng)
    nom_x, nom_y = _by_class(torch, model, 100, rng)
    ood_x, ood_y = _by_class(torch, model, 80, rng, scale=1.3)
    out = str(tmp_path_factory.mktemp("out"))
    active, apfds = {}, {}
    torch.manual_seed(1)
    for model_id in MODEL_IDS:
        np.random.seed(SEED + model_id)
        active[model_id] = AL.evaluate(model_id, CASE_STUDY, model, train_x, train_y, nom_x, nom_y, ood_x, ood_y,
                                       nc_activation_layers=NC_LAYERS, sa_activation_layers=SA_LAYERS,
                                       training_process=_training_process(torch, model), observed_share=SHARE,
                                       num_selected=NUM_SELECTED, num_classes=3, output_folder=out)
        apfds[model_id] = P.evaluate(model_id, CASE_STUDY, model, train_x, nom_x, nom_y, ood_x, ood_y,
                                     nc_activation_layers=NC_LAYERS, sa_activation_layers=SA_LAYERS,
                                     output_folder=out)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")              # the runs 2..99 every approach misses
        written = {t: E.evaluate_results(out, t, [CASE_STUDY]) for t in E.EVAL_TYPES}
    return out, active, apfds, written


def _fmt(x):
    return f"{x:.2%}"


def test_active_learning_table_equals_the_returned_accuracies(run):
    import pandas as pd
    from simple_tip_b200.core import results as R

    out, active, _, written = run
    assert written["active_learning"] == [os.path.join(out, "results", "active.csv")]
    df = pd.read_csv(written["active_learning"][0], header=[0, 1, 2], index_col=[0, 1])
    assert list(df.index) == [(R.category(a), a) for a in ["original", "random"] + R.APPROACHES]
    assert len(active[0][1]) == 2 * (len(R.APPROACHES) + 1)
    for active_split in SPLITS:
        for key in active[0][0]:
            col = (CASE_STUDY, active_split, f"{key[0]}:{key[1]}")
            original = (active[0][0][key] + active[1][0][key]) / 2
            assert df.loc[("baseline", "original"), col] == _fmt(original), col
            random = (active[0][2][("random", active_split)][key] + active[1][2][("random", active_split)][key]) / 2
            assert df.loc[("baseline", "random"), col] == _fmt(random), col
            for approach in R.APPROACHES:
                mean = sum(active[i][2][(approach, active_split)][key] for i in MODEL_IDS) / 2
                assert df.loc[(R.category(approach), approach), col] == _fmt(mean - random), (approach, col)


def _a12_grid(values, approaches):
    """A12 of every pair i < j of {approach: [value of model 0, value of model 1]}, NaN for equal pairs."""
    n = len(approaches)
    e = np.full((n, n), -10000.0)
    for i in range(n):
        for j in range(i + 1, n):
            x, y = np.array(values[approaches[i]]), np.array(values[approaches[j]])
            if np.array_equal(x, y):
                e[i, j] = np.nan
            else:
                e[i, j] = 2 * abs(((x > y).sum() + 0.5 * (x == y).sum()) / x.size - 0.5)
    return e


def _read_statistics(paths):
    import pandas as pd

    p, e = (pd.read_csv(path, index_col=0) for path in paths)
    assert p.shape == e.shape == (39, 39)
    assert list(p.index) == list(p.columns) == list(e.index) == list(e.columns)
    return p, e


def test_statistics_effect_sizes_equal_a12_of_the_ood_values(run):
    from simple_tip_b200.core import results as R

    out, active, apfds, written = run
    results = os.path.join(out, "results")
    for eval_type, values, name in (
            ("test_prio_statistics", {a: [apfds[i]["ood"][a] for i in MODEL_IDS] for a in R.APPROACHES}, "apfd"),
            ("active_learning_statistics",
             {a: [active[i][2][(a, "ood")][("ood", "future")] for i in MODEL_IDS] for a in R.APPROACHES}, "active")):
        assert written[eval_type] == [os.path.join(results, f"{name}_correlation_{k}.csv") for k in ("p", "eff")]
        p, e = _read_statistics(written[eval_type])
        want = _a12_grid(values, R.APPROACHES)
        np.testing.assert_array_equal(e.to_numpy(dtype=np.float64), want, err_msg=eval_type)
        upper = np.triu(np.ones(want.shape, dtype=bool), 1)
        p = p.to_numpy(dtype=np.float64)
        assert np.isnan(p[~upper]).all()                       # the fill written as empty cells
        assert np.array_equal(np.isnan(p[upper]), np.isnan(want[upper]))
        ok = ~np.isnan(p) & upper
        assert ok.any() and ((p[ok] > 0) & (p[ok] <= 1)).all()


def test_every_file_reads_back(run):
    import pandas as pd

    out, _, _, written = run
    files = sorted(p for paths in written.values() for p in paths)
    assert files == sorted(os.path.join(out, "results", f) for f in os.listdir(os.path.join(out, "results")))
    assert len(files) == 6
    for path in files:
        assert not pd.read_csv(path, header=None).empty, path
