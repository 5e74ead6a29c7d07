"""Training a stack of models on the GPU: `tip_softmax_xent_seg` segment by segment against `tip_softmax_xent`,
`tip_stack_gather` against torch indexing, `fit_stack` against `_fit` model by model, a stack learning a learnable
task, active learning's stacked retraining against its sequential loop, and the runner with stacked=True."""
import copy
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    import torch

    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---- the kernels ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("classes", [2, 10, 32])
@pytest.mark.parametrize("rows", [1, 33, 128])
@pytest.mark.parametrize("segments", [1, 3, 80])
def test_softmax_xent_seg_equals_each_segment_alone(segments, rows, classes):
    import torch

    from simple_tip_b200 import engine as E

    g = torch.Generator(device="cuda").manual_seed(segments * 1000 + rows * 10 + classes)
    z = torch.randn((segments, rows, classes), device="cuda", generator=g) * 4.0
    y = torch.nn.functional.one_hot(torch.randint(0, classes, (segments, rows), device="cuda", generator=g),
                                    classes).float()
    y[0, 0] = 1.0 / classes                               # one soft target row
    loss, correct = torch.empty(segments, device="cuda"), torch.empty(segments, dtype=torch.int32, device="cuda")
    dz = torch.empty_like(z)
    E.softmax_xent_seg(z, y, loss, dz, correct)
    loss_nodz, correct_nodz = torch.empty_like(loss), torch.empty_like(correct)
    E.softmax_xent_seg(z, y, loss_nodz, None, correct_nodz)
    for s in range(segments):
        l1, c1 = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
        d1 = torch.empty((rows, classes), device="cuda")
        E.softmax_xent(z[s], y[s], l1, d1, c1)
        assert torch.equal(loss[s:s + 1], l1) and torch.equal(correct[s:s + 1], c1), s
        assert torch.equal(dz[s], d1), s
        assert torch.equal(loss_nodz[s:s + 1], l1) and torch.equal(correct_nodz[s:s + 1], c1), s


def _gather_want(torch, pool, rows, perm, start, b, interleaved):
    idx = torch.gather(rows, 1, perm[:, start:start + b])            # [M, b]
    got = pool[idx]                                                  # [M, b, ...]
    if pool.dtype == torch.float64:
        got = got.float()
    if interleaved:                                                  # [M, b, H, W, C] -> [b, H, W, M * C]
        m, b_, h, w, c = got.shape
        got = got.permute(1, 2, 3, 0, 4).reshape(b_, h, w, m * c)
    return got.contiguous()


@pytest.mark.parametrize("m", [1, 5])
@pytest.mark.parametrize("dtype", ["float32", "float64", "int32"])
def test_stack_gather_equals_torch_indexing(m, dtype):
    import torch

    from simple_tip_b200 import engine as E

    g = torch.Generator(device="cuda").manual_seed(m)
    n_pool, n_rows, n_perm = 300, 70, 61
    shapes = {"float32": [(8, 8, 3), (10,)], "float64": [(6, 6, 3)], "int32": [(100,)]}[dtype]
    rows = torch.randint(0, n_pool, (m, n_rows), device="cuda", generator=g)
    perm = torch.stack([torch.randperm(n_perm, device="cuda", generator=g) for _ in range(m)])
    for shape in shapes:
        pool = (torch.randint(-5000, 5000, (n_pool, *shape), device="cuda", generator=g).to(getattr(torch, dtype))
                if dtype == "int32" else torch.randn((n_pool, *shape), device="cuda", generator=g,
                                                     dtype=getattr(torch, dtype)) * 3)
        for interleaved in ((False, True) if len(shape) == 3 else (False,)):
            for start, b in ((0, 16), (48, 13), (0, n_perm)):            # full, partial last batch, everything
                got = E.stack_gather(pool, rows, perm, start, b, interleaved)
                want = _gather_want(torch, pool, rows, perm, start, b, interleaved)
                assert got.dtype == want.dtype and got.shape == want.shape
                assert torch.equal(got, want), (shape, interleaved, start, b)
                out = torch.full_like(got, 9)
                assert E.stack_gather(pool, rows, perm, start, b, interleaved, out=out, check=False) is out
                assert torch.equal(out, want)


def test_stack_gather_refusals():
    import torch

    from simple_tip_b200 import engine as E

    rows = torch.zeros((2, 4), dtype=torch.int64, device="cuda")
    perm = torch.arange(4, device="cuda").expand(2, 4).contiguous()
    for dtype in (torch.float16, torch.uint8, torch.int64):
        with pytest.raises(ValueError, match="float32, float64 or int32"):
            E.stack_gather(torch.zeros((10, 3), dtype=dtype, device="cuda"), rows, perm, 0, 4)
    pool = torch.zeros((10, 3), device="cuda")
    for bad in (10, -1):
        r = rows.clone()
        r[1, 2] = bad
        with pytest.raises(ValueError, match="outside the pool"):
            E.stack_gather(pool, r, perm, 0, 4)
    with pytest.raises(ValueError):
        E.stack_gather(pool, rows, perm, 2, 3)                      # past the permutation's end
    with pytest.raises(ValueError):
        E.stack_gather(pool, rows.int(), perm, 0, 4)


# ---- fit_stack against fit -------------------------------------------------------------------------------------------
def _no_dropout(model):
    import torch

    for layer in model.modules():
        if isinstance(layer, torch.nn.Dropout):
            layer.p = 0.0
    return model


def _pool(torch, name, n):
    g = torch.Generator().manual_seed(len(name) + n)
    if name == "imdb":
        x = torch.randint(1, 2000, (n, 100), generator=g, dtype=torch.int32)
        x[:, :40] = 0
        classes = 2
    elif name == "cifar10":
        x, classes = torch.rand((n, 32, 32, 3), generator=g, dtype=torch.float64), 10
    else:
        x, classes = torch.rand((n, 28, 28, 1), generator=g), 10
    labels = torch.randint(0, classes, (n,), generator=g)
    return x.cuda(), torch.nn.functional.one_hot(labels, classes).float().cuda()


@pytest.mark.parametrize("name", ["mnist", "cifar10", "imdb"])
def test_fit_stack_equals_fit_model_by_model(name):
    import torch

    from simple_tip_b200.case_studies import CASE_STUDIES
    from simple_tip_b200.core import training

    network = CASE_STUDIES[name].network
    x, y = _pool(torch, name, 300)
    m, n_rows, batch, seeds = 3, 40, 64, [3, 8, 21]
    g = torch.Generator().manual_seed(5)
    rows = torch.stack([torch.randperm(300, generator=g)[:n_rows] for _ in range(m)]).cuda()
    # 40 rows, 4 held out: 36 training rows, one full-batch step per epoch, so the shuffle only reorders sums
    models = training.fit_stack([_no_dropout(network().cuda()) for _ in range(m)], x, y, rows, batch, 3, 0.1,
                                seeds=seeds)
    assert len(models) == m
    for k, (model, seed) in enumerate(zip(models, seeds)):
        assert not model.training
        ref = training._fit(_no_dropout(network().cuda()), x[rows[k]], y[rows[k]], batch, 3, 0.1, seed, graph=False)
        for key in ("loss", "accuracy", "val_loss", "val_accuracy"):
            assert len(model.history[key]) == 3, key
        assert model.history["loss"] == pytest.approx(ref.history["loss"], rel=1e-5), k
        assert model.history["val_loss"] == pytest.approx(ref.history["val_loss"], rel=1e-5), k
        # Adam divides each gradient by its own running magnitude, so where a gradient element nearly cancels, a
        # rounding-level difference (grouped against single convolutions) moves its parameter by a share of the
        # step size lr = 1e-3 rather than by a share of the parameter: every element stays within one step, and
        # the median element within 1e-4 of the tensor's largest magnitude (1e-6 absolute for tensors whose gradient
        # is zero but for rounding, as the attention's key bias)
        for (pname, a), b in zip(model.named_parameters(), ref.parameters()):
            err, scale = torch.abs(a - b).detach().flatten().double(), float(torch.max(torch.abs(b)))
            assert float(err.max()) <= training.ADAM["lr"], (k, pname, float(err.max()))
            bulk = float(torch.median(err))
            assert bulk <= max(1e-4 * scale, 1e-6), (k, pname, bulk, scale)


# ---- learning ----------------------------------------------------------------------------------------------------------
def _blocks(rng, n):
    """MNIST-shaped uint8 images whose class is the 7 x 7 block (of a 4 x 4 grid) that is bright."""
    labels = rng.integers(0, 10, size=n)
    x = rng.integers(0, 90, size=(n, 28, 28), dtype=np.uint8)
    for i, c in enumerate(labels):
        r, k = divmod(int(c), 4)
        x[i, 7 * r:7 * r + 7, 7 * k:7 * k + 7] += np.uint8(160)
    return x, labels.astype(np.uint8)


def _tensors(torch, x, labels):
    xt = torch.from_numpy(np.expand_dims(x, -1).astype(np.float32) / 255.0).cuda()
    yt = torch.nn.functional.one_hot(torch.from_numpy(labels.astype(np.int64)).cuda(), 10).float()
    return xt, yt


def test_a_stack_learns_a_learnable_task():
    import torch

    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import active_learning, training

    rng = np.random.default_rng(1)
    x, labels = _blocks(rng, 6000)
    xt, yt = _tensors(torch, x, labels)
    g = torch.Generator().manual_seed(2)
    rows = torch.stack([torch.randperm(6000, generator=g)[:5000] for _ in range(4)]).cuda()
    models = training.fit_stack([mnist.network().cuda() for _ in range(4)], xt, yt, rows, 128, 2,
                                seeds=[0, 1, 2, 3])
    hx, hl = _blocks(rng, 1000)
    hxt = _tensors(torch, hx, hl)[0]
    for model in models:
        acc = active_learning.accuracy(model, hxt, torch.from_numpy(hl.astype(np.int64)).cuda())
        assert acc >= 0.95, acc
        assert not model.training and len(model.history["val_accuracy"]) == 2
    params = [torch.cat([p.flatten() for p in model.parameters()]) for model in models]
    assert all(not torch.equal(params[i], params[j]) for i in range(4) for j in range(i + 1, 4))


# ---- active learning -------------------------------------------------------------------------------------------------
NC_LAYERS, SA_LAYERS = [0, 2, 4], [4]
NUM_SELECTED, SHARE, MODEL_ID, SEED = 20, 0.5, 5, 2024


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
    x = torch.from_numpy((rng.normal(size=(pool, 1, 12, 12)) * scale).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x)
    top = z.topk(2, dim=1).values
    pred = z.argmax(dim=1).cpu().numpy()
    clear = ((top[:, 0] - top[:, 1]) > 1e-3).cpu().numpy()
    rows = np.concatenate([np.flatnonzero((pred == c) & clear)[:per_class] for c in range(3)])
    return x[torch.from_numpy(rows).cuda()], torch.from_numpy(pred[rows].astype(np.int64)).cuda()


def _fake(torch, model, y):
    """The deterministic retraining of the sequential spy: the model with its last bias moved by the labels at the
    head of its data."""
    m = copy.deepcopy(model)
    with torch.no_grad():
        m[-2].bias += (y[:64].sum(dim=0).to(m[-2].bias.device) / 64 - 1 / 3) * 4.0
    return m


@pytest.fixture(scope="module")
def al_runs(tmp_path_factory):
    import torch

    from simple_tip_b200.core import active_learning as AL

    model = _toy_model(torch)
    rng = np.random.default_rng(0)
    train_x, train_y = _by_class(torch, model, 150, rng)
    nom_x, nom_y = _by_class(torch, model, 100, rng)
    ood_x, ood_y = _by_class(torch, model, 80, rng, scale=1.3)
    data = {"train_x": train_x, "train_y": train_y, "nominal_test_x": nom_x, "nominal_test_labels": nom_y,
            "ood_test_x": ood_x, "ood_test_labels": ood_y}
    handed, stacked_calls = [], []

    def training_process(x, y):
        handed.append((x.clone(), y.clone()))
        return _fake(torch, model, y)

    def stacked_training_process(x_pool, y_pool, rows):
        stacked_calls.append((x_pool, y_pool, rows))
        return [_fake(torch, model, y_pool[r]) for r in rows]
    res = {}
    for name, kwargs in (("sequential", dict(training_process=training_process)),
                         ("stacked", dict(training_process=None, stacked_training_process=stacked_training_process))):
        out = tmp_path_factory.mktemp(name)
        np.random.seed(SEED)
        res[name] = (AL.evaluate(MODEL_ID, "toy", model, nc_activation_layers=NC_LAYERS, sa_activation_layers=SA_LAYERS,
                                 observed_share=SHARE, num_selected=NUM_SELECTED, num_classes=3,
                                 output_folder=str(out), **data, **kwargs), str(out))
    return handed, stacked_calls, res


def test_stacked_rows_give_the_sequential_handed_over_data(al_runs):
    import torch

    handed, stacked_calls, _ = al_runs
    assert len(stacked_calls) == 1
    x_pool, y_pool, rows = stacked_calls[0]
    assert rows.dtype == torch.int64 and rows.device == x_pool.device == y_pool.device
    assert rows.shape == (len(handed), handed[0][0].shape[0]) == (80, 450 + NUM_SELECTED)
    assert x_pool.shape[0] == 450 + 150 + 120 and y_pool.dtype == torch.float32
    for k, (x, y) in enumerate(handed):
        assert torch.equal(x_pool[rows[k]], x), k
        assert torch.equal(y_pool[rows[k]], y), k


def test_stacked_results_and_files_equal_the_sequential_run(al_runs):
    _, _, res = al_runs
    (seq, seq_dir), (stk, stk_dir) = res["sequential"], res["stacked"]
    assert seq[0] == stk[0]
    assert list(seq[1]) == list(stk[1])
    for key in seq[1]:
        np.testing.assert_array_equal(np.asarray(seq[1][key]), np.asarray(stk[1][key]))
    assert list(seq[2].items()) == list(stk[2].items())
    files = sorted(os.listdir(os.path.join(seq_dir, "active_learning")))
    assert files and files == sorted(os.listdir(os.path.join(stk_dir, "active_learning")))
    for f in files:
        with open(os.path.join(seq_dir, "active_learning", f), "rb") as a, \
                open(os.path.join(stk_dir, "active_learning", f), "rb") as b:
            assert a.read() == b.read(), f


# ---- the runner ----------------------------------------------------------------------------------------------------------
def test_runner_trains_and_retrains_in_stacks(tmp_path, monkeypatch):
    import torch

    from simple_tip_b200.case_studies import load_model, mnist
    from simple_tip_b200.core import evaluation

    for k, v in {"B200TIP_KDE": "device", "B200TIP_COV": "device", "B200TIP_GMM": "device",
                 "B200TIP_KMEANS": "device"}.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(2)
    nominal = (_blocks(rng, 3000), _blocks(rng, 300))
    data = tmp_path / "datasets"
    data.mkdir()
    cx, cl = _blocks(rng, 300)
    np.save(data / "mnist_c_images.npy", np.expand_dims(255 - cx, -1))
    np.save(data / "mnist_c_labels.npy", cl.astype(np.int64))
    datasets = mnist.load_datasets(nominal, str(data))
    outs = {}
    for stacked in (False, True):
        out = str(tmp_path / f"assets_{stacked}")
        cs = mnist.MnistCaseStudy(out, datasets, epochs=1, num_selected=20)
        np.random.seed(0)
        cs.train([0, 1, 2], stacked=stacked)
        for i in (0, 1, 2):
            model = load_model(out, "mnist", i)
            assert all(torch.isfinite(p).all() for p in model.parameters())
        cs.run_active_learning_eval([0], stacked=stacked)
        outs[stacked] = sorted(os.listdir(os.path.join(out, "active_learning")))
        al = evaluation.active_learning_table(out, ["mnist"])
        assert al.shape[0] > 0
    assert outs[True] == outs[False] and outs[True]
