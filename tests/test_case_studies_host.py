"""The case studies' networks, initialisers, datasets and layer choices on the host (no GPU needed)."""
import math

import numpy as np
import pytest
import torch

from simple_tip_b200.case_studies import cifar10, fmnist, imdb, mnist
from simple_tip_b200.core import imdb as imdb_inputs
from simple_tip_b200.core.training import glorot_limit, keras_fans, keras_initialize, validation_rows

IMAGE = (2, 28, 28, 1)
CASES = {
    # name: (network, input shape, per-child output shapes, parameters)
    "mnist": (mnist.network, IMAGE, [(2, 26, 26, 32), (2, 13, 13, 32), (2, 11, 11, 64), (2, 5, 5, 64), (2, 1600),
                                     (2, 1600), (2, 10)], 34826),
    "fmnist": (fmnist.network, IMAGE, [(2, 26, 26, 32), (2, 13, 13, 32), (2, 11, 11, 64), (2, 5, 5, 64), (2, 1600),
                                       (2, 1600), (2, 10)], 34826),
    "cifar10": (cifar10.network, (2, 32, 32, 3), [(2, 30, 30, 32), (2, 15, 15, 32), (2, 13, 13, 64), (2, 6, 6, 64),
                                                  (2, 4, 4, 64), (2, 1024), (2, 64), (2, 10)], 122570),
    "imdb": (imdb.network, (2, 100), [(2, 100), (2, 100, 32), (2, 100, 32), (2, 32), (2, 32), (2, 20), (2, 20),
                                      (2, 2)], 78558),
}


def _input(name, shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    if name == "imdb":
        return torch.randint(0, imdb_inputs.VOCAB_SIZE, shape, generator=g, dtype=torch.int32)
    return torch.rand(shape, generator=g)


@pytest.mark.parametrize("name", sorted(CASES))
def test_children_are_keras_layers_with_keras_shapes(name):
    network, shape, child_shapes, n_params = CASES[name]
    net = network().eval()
    outs = []
    for c in net.children():
        c.register_forward_hook(lambda _m, _i, o: outs.append(o))
    with torch.no_grad():
        y = net(_input(name, shape))
    assert [tuple(o.shape) for o in outs] == child_shapes
    assert sum(p.numel() for p in net.parameters()) == n_params
    assert torch.allclose(y.sum(dim=1), torch.ones(2), atol=1e-6)
    with torch.no_grad():
        assert torch.allclose(torch.softmax(net.logits(_input(name, shape)), dim=1), y, atol=1e-6)


def test_image_layers_hand_nhwc_in_flatten_order():
    net = mnist.network().eval()
    traces = []
    for i in (3, 4):
        list(net.children())[i].register_forward_hook(lambda _m, _i, o: traces.append(o))
    with torch.no_grad():
        net(_input("mnist", IMAGE))
    pooled, flat = traces
    assert torch.equal(flat, pooled.reshape(2, -1))          # Keras' Flatten of (H, W, C)


def test_keras_fans():
    assert keras_fans((3, 3, 32, 64)) == (9 * 32, 9 * 64)     # Conv2D kernel (kh, kw, in, out)
    assert keras_fans((1600, 10)) == (1600, 10)
    assert keras_fans((32, 2, 32)) == (2 * 32, 32 * 32)      # attention projection [embed, heads, key_dim]
    assert keras_fans((2, 32, 32)) == (32 * 2, 32 * 2)       # attention output [heads, key_dim, embed]


@pytest.mark.parametrize("name", sorted(CASES))
def test_keras_initialisers(name):
    net = keras_initialize(CASES[name][0](), torch.Generator().manual_seed(3))
    seen = 0
    for mod_name, p in net.named_parameters():
        leaf = mod_name.rsplit(".", 1)[-1]
        if leaf in ("bias",) or leaf.endswith("_bias"):
            if "layernorm" in mod_name:
                continue
            assert torch.count_nonzero(p) == 0, mod_name
        elif leaf in ("token_emb", "pos_emb"):
            assert p.abs().max() <= 0.05 and p.abs().max() > 0.04, mod_name
        elif "layernorm" in mod_name:
            assert torch.all(p == 1), mod_name
        else:
            shape = tuple(p.shape)
            if p.dim() == 4:                                   # torch's conv layout -> Keras' (kh, kw, in, out)
                shape = (shape[2], shape[3], shape[1], shape[0])
            limit = glorot_limit(shape)
            assert p.abs().max() <= limit and p.abs().max() > 0.9 * limit, mod_name
            seen += 1
    assert seen >= 3
    again = keras_initialize(CASES[name][0](), torch.Generator().manual_seed(3))
    assert all(torch.equal(a, b) for a, b in zip(net.parameters(), again.parameters()))


def test_attention_kernels_use_keras_fans():
    att = imdb.network()[2].att
    assert att.query_kernel.shape == (32, 2, 32) and att.output_kernel.shape == (2, 32, 32)
    assert glorot_limit(att.query_kernel.shape) == pytest.approx(math.sqrt(6.0 / (64 + 1024)))


@pytest.mark.parametrize("n, split, held_out", [(60000, 0.1, 6000), (1001, 0.1, 101), (10, 0.1, 1), (7, 0.1, 1),
                                                (25000, 0.1, 2500), (3, 0.5, 2), (5, 0.0, 0)])
def test_validation_rows(n, split, held_out):
    assert validation_rows(n, split) == held_out == n - int(math.floor(n * (1.0 - split)))


def test_effective_imdb_nc_layers():
    # handler_model.py:198-202: `layer for i, layer in enumerate(model.layers) if i in activation_layers`
    ref = [i for i, _ in enumerate(range(8)) if i in imdb.REFERENCE_NC_ACTIVATION_LAYERS]
    assert imdb.NC_ACTIVATION_LAYERS == ref == [3, 5]
    assert imdb.ImdbCaseStudy.sa_layers == [5] and imdb.ImdbCaseStudy.dsa_badge_size == 500


# ---- datasets: the reference's expressions restated on small synthetic arrays ----------------------------------
def _nominal(rng, shape, labels_2d=False):
    def labels(n):
        y = rng.integers(0, 10, size=n).astype(np.uint8)
        return y.reshape(-1, 1) if labels_2d else y
    return ((rng.integers(0, 256, size=(40,) + shape, dtype=np.uint8), labels(40)),
            (rng.integers(0, 256, size=(12,) + shape, dtype=np.uint8), labels(12)))


def _equal(a, b):
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v)


def test_mnist_datasets(tmp_path):
    rng = np.random.default_rng(0)
    nominal = _nominal(rng, (28, 28))
    np.save(tmp_path / "mnist_c_images.npy", rng.integers(0, 256, size=(9, 28, 28, 1), dtype=np.uint8))
    np.save(tmp_path / "mnist_c_labels.npy", rng.integers(0, 10, size=9).astype(np.int64))
    (x_train, y_train), (x_test, y_test) = nominal
    x_test = np.expand_dims(x_test, -1).astype("float32") / 255.0
    x_train = np.expand_dims(x_train, -1).astype("float32") / 255.0
    ood_x = np.load(tmp_path / "mnist_c_images.npy").astype("float32") / 255.0
    ood_y = np.load(tmp_path / "mnist_c_labels.npy")
    ood_x, ood_y = np.concatenate((x_test, ood_x), axis=0), np.concatenate((y_test, ood_y), axis=0)
    p = np.random.default_rng(0).permutation(len(ood_y))
    want = ((x_train, y_train), (x_test, y_test), (ood_x[p], ood_y[p]))
    got = mnist.load_datasets(nominal, str(tmp_path))
    _equal(got, want)
    assert got[0][0].dtype == np.float32


def test_fmnist_datasets(tmp_path):
    rng = np.random.default_rng(1)
    nominal = _nominal(rng, (28, 28))
    np.save(tmp_path / "fmnist-c-test.npy", rng.integers(0, 256, size=(9, 28, 28), dtype=np.uint8))
    np.save(tmp_path / "fmnist-c-test-labels.npy", rng.integers(0, 10, size=9).astype(np.uint8))
    (x_train, y_train), (x_test, y_test) = nominal
    x_test = np.expand_dims(x_test, -1).astype("float32") / 255.0
    x_train = np.expand_dims(x_train, -1).astype("float32") / 255.0
    ood_x = np.load(tmp_path / "fmnist-c-test.npy").astype("float32") / 255.0
    ood_y = np.load(tmp_path / "fmnist-c-test-labels.npy")
    ood_x = np.concatenate((x_test, np.expand_dims(ood_x, -1)), axis=0)
    ood_y = np.concatenate((y_test, ood_y), axis=0)
    p = np.random.default_rng(0).permutation(len(ood_y))
    _equal(fmnist.load_datasets(nominal, str(tmp_path)), ((x_train, y_train), (x_test, y_test), (ood_x[p], ood_y[p])))


def test_cifar10_c_and_datasets(tmp_path):
    rng = np.random.default_rng(2)
    src, out = tmp_path / "CIFAR-10-C", tmp_path / "datasets"
    src.mkdir()
    labels = rng.integers(0, 10, size=6).astype(np.uint8)
    np.save(src / "labels.npy", labels)
    files = {}
    for name in ("zoom_blur.npy", "brightness.npy", "fog.npy"):
        files[name] = rng.integers(0, 256, size=(6, 32, 32, 3), dtype=np.uint8)
        np.save(src / name, files[name])
    (src / "README.txt").write_text("not an array")
    cifar10.prepare_cifar10_c(str(src), str(out))
    order = sorted(files)
    allc = np.concatenate([files[f] for f in order], axis=0)
    idx = np.random.default_rng(0).permutation(len(allc))[:10000]
    assert np.array_equal(np.load(out / "cifar10_c_images.npy"), allc[idx])
    assert np.array_equal(np.load(out / "cifar10_c_labels.npy"), np.tile(labels, len(order))[idx])

    nominal = _nominal(rng, (32, 32, 3), labels_2d=True)
    (x_train, y_train), (x_test, y_test) = nominal
    x_train, x_test = x_train / 255.0, x_test / 255.0
    y_test, y_train = y_test.flatten(), y_train.flatten()
    ood_x = np.load(out / "cifar10_c_images.npy").astype("float32") / 255.0
    ood_y = np.load(out / "cifar10_c_labels.npy")
    ood_x = np.concatenate((x_test, ood_x), axis=0)
    ood_y = np.concatenate((y_test.flatten(), ood_y), axis=0)
    p = np.random.default_rng(0).permutation(len(ood_y))
    got = cifar10.load_datasets(nominal, str(out))
    _equal(got, ((x_train, y_train), (x_test, y_test), (ood_x[p], ood_y[p])))
    assert got[0][0].dtype == np.float64 and got[2][0].dtype == np.float64


def test_cifar10_c_needs_the_folder(tmp_path):
    with pytest.raises(FileNotFoundError, match="CIFAR-10-C"):
        cifar10.prepare_cifar10_c(str(tmp_path / "missing"), str(tmp_path / "out"))


def test_case_study_constants():
    for cs, bs, ep, sel in ((mnist.MnistCaseStudy, 128, 15, 1000), (fmnist.FashionMnistCaseStudy, 128, 15, 1000),
                            (cifar10.Cifar10CaseStudy, 32, 20, 1000), (imdb.ImdbCaseStudy, 32, 10, 2500)):
        assert (cs.batch_size, cs.epochs, cs.num_selected) == (bs, ep, sel)
    assert imdb.load_datasets is imdb_inputs.load_datasets
