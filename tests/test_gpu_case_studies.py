"""The case studies on the GPU: graph-captured `fit` against an eager replay of the same steps, learning a learnable
task, the MNIST-shaped runner through all four phases into one folder, and the IMDB network's training and traces."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DEVICE_BACKENDS = {"B200TIP_KDE": "device", "B200TIP_COV": "device", "B200TIP_GMM": "device",
                   "B200TIP_KMEANS": "device"}


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


def test_graph_steps_equal_an_eager_replay():
    import torch

    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import training

    x, labels = _blocks(np.random.default_rng(0), 1000)
    xt, yt = _tensors(torch, x, labels)
    models = []
    for graph in (True, False):
        net = mnist.network().cuda()
        for m in net.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        # 900 training rows in batches of 64: 14 full steps and a tail of 4 per epoch, 30 steps in two epochs
        models.append(training._fit(net, xt, yt, 64, 2, 0.1, seed=11, graph=graph))
    for (name, a), b in zip(models[0].named_parameters(), models[1].parameters()):
        assert torch.max(torch.abs(a - b)) <= 1e-5 * torch.max(torch.abs(b)), name
    assert models[0].history["loss"] == pytest.approx(models[1].history["loss"], rel=1e-5)
    assert len(models[0].history["val_accuracy"]) == 2


def test_fit_learns_a_learnable_task():
    import torch

    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import active_learning, training

    rng = np.random.default_rng(1)
    x, labels = _blocks(rng, 6000)
    xt, yt = _tensors(torch, x, labels)
    model = training.fit(mnist.network().cuda(), xt, yt, 128, 2, seed=0)
    hx, hl = _blocks(rng, 1000)
    acc = active_learning.accuracy(model, _tensors(torch, hx, hl)[0], torch.from_numpy(hl.astype(np.int64)).cuda())
    assert acc >= 0.95, acc
    assert not model.training


def test_mnist_case_study_runs_every_phase(tmp_path, monkeypatch):
    import torch

    from simple_tip_b200.case_studies import load_model, mnist
    from simple_tip_b200.core import activations, evaluation, results

    for k, v in DEVICE_BACKENDS.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(2)
    nominal = (_blocks(rng, 6000), _blocks(rng, 300))
    data = tmp_path / "datasets"
    data.mkdir()
    cx, cl = _blocks(rng, 300)
    np.save(data / "mnist_c_images.npy", np.expand_dims(255 - cx, -1))
    np.save(data / "mnist_c_labels.npy", cl.astype(np.int64))
    out = str(tmp_path / "assets")
    cs = mnist.MnistCaseStudy(out, mnist.load_datasets(nominal, str(data)), epochs=2, num_selected=20)

    np.random.seed(0)
    cs.train([0, 1])
    for i in (0, 1):
        assert os.path.exists(os.path.join(out, "models", "mnist", f"model_{i}.pt"))
    apfds = cs.run_prio_eval([0, 1])
    assert set(apfds) == {0, 1} and set(apfds[0]) == {"nominal", "ood"}
    table = results.apfd_table(out, ["mnist"])
    assert table.shape[0] > 0
    cs.run_active_learning_eval([0])
    assert os.listdir(os.path.join(out, "active_learning"))
    al = evaluation.active_learning_table(out, ["mnist"])
    assert al.shape[0] > 0

    cs.collect_activations([1])
    model = load_model(out, "mnist", 1)
    n_layers = len(list(model.children()))
    tm = activations.TransparentModel(model, list(range(n_layers)), include_last_layer=False)
    for ds, (x, y) in (("train", cs.train_set), ("test_nominal", cs.nominal_set),
                       ("test_nominal_and_corrupted", cs.ood_set)):
        acts, lab = activations.load_badges(out, "mnist", 1, ds)
        assert len(acts) == n_layers and np.array_equal(lab, y)
        want = tm.collect(x, activations.BADGE_SIZE)
        assert acts[3].shape == (x.shape[0], 5, 5, 64)
        for a, w in zip(acts, want):
            assert np.array_equal(a, w.cpu().numpy())
    assert all(torch.equal(a, b) for a, b in zip(model.parameters(), cs.load_model(1).parameters()))


def test_imdb_trains_and_traces_with_keras_shapes():
    import torch

    from simple_tip_b200.case_studies import imdb
    from simple_tip_b200.core import activations, training

    rng = np.random.default_rng(3)
    n = 1000
    labels = rng.integers(0, 2, size=n)
    ids = rng.integers(1, 2000, size=(n, 100)).astype(np.int32)
    ids[:, :40] = 0                                            # pre-padding, as pad_sequences leaves it
    ids[:, 50] = np.where(labels == 1, 7, 9)                   # a word that gives the class away
    x = torch.from_numpy(ids).cuda()
    y = torch.nn.functional.one_hot(torch.from_numpy(labels).cuda(), 2).float()
    model = training.fit(imdb.network().cuda(), x, y, imdb.ImdbCaseStudy.batch_size, 1, seed=4)
    assert len(model.history["loss"]) == 1 and np.isfinite(model.history["loss"][0])
    tm = activations.TransparentModel(model, list(range(8)), include_last_layer=True)
    acts = tm.get_activations(x[:5])
    assert [tuple(a.shape) for a in acts] == [(5, 100), (5, 100, 32), (5, 100, 32), (5, 32), (5, 32), (5, 20),
                                              (5, 20), (5, 2), (5, 2)]
    assert torch.allclose(acts[-1].sum(dim=1), torch.ones(5, device="cuda"), atol=1e-6)
