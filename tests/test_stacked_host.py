"""The stacked networks of `case_studies.stacked` on the CPU: each model's slice of the stacked logits against the
model's own logits for all four case-study networks, stack -> unstack bit for bit, the refusals, and seeded
re-initialisation."""
import pytest
import torch

from simple_tip_b200.case_studies import cifar10, fmnist, imdb, mnist, stacked
from simple_tip_b200.case_studies.base import Dense, KerasSequential
from simple_tip_b200.core.training import keras_initialize


def _images(shape, dtype=torch.float32):
    return lambda g: torch.rand(shape, generator=g, dtype=dtype)


def _ids(g):
    ids = torch.randint(1, 2000, (6, 100), generator=g, dtype=torch.int32)
    ids[:, :30] = 0                                            # pre-padding, as pad_sequences leaves it
    return ids


NETWORKS = {
    "mnist": (mnist.network, _images((6, 28, 28, 1))),
    "fmnist": (fmnist.network, _images((6, 28, 28, 1))),
    "cifar10": (cifar10.network, _images((6, 32, 32, 3), torch.float64)),       # load_datasets' float64 images
    "imdb": (imdb.network, _ids),                                               # int32 token ids
}


def _models(network, m, seed=0):
    torch.manual_seed(seed)
    models = [network() for _ in range(m)]
    for model in models:
        for layer in model.modules():
            if isinstance(layer, torch.nn.Dropout):
                layer.p = 0.0
    return models


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("m", [1, 3])
@pytest.mark.parametrize("name", sorted(NETWORKS))
def test_stacked_logits_equal_each_models_own(name, m, mode):
    network, inputs = NETWORKS[name]
    models = _models(network, m)
    for model in models:
        model.train(mode == "train")
    net = stacked.stack(models)
    assert net.training == (mode == "train")
    g = torch.Generator().manual_seed(1)
    xs = [inputs(g) for _ in range(m)]
    with torch.no_grad():
        z = net.logits(net.stack_inputs(xs))
        assert z.shape == (m, 6, models[0][-1].kernel.shape[1]) and z.is_contiguous()
        for k, (model, x) in enumerate(zip(models, xs)):
            want = model.logits(x)
            torch.testing.assert_close(z[k], want, rtol=1e-5, atol=1e-5 * float(want.abs().max()))
            if m == 1 and name != "imdb":
                assert torch.equal(z[k], want)
            probs = net(net.stack_inputs(xs))[k]
            torch.testing.assert_close(probs, model(x), rtol=1e-5, atol=1e-6)


def test_interleaved_layout_only_for_image_stacks():
    assert stacked.stack(_models(mnist.network, 2)).channels_interleaved
    assert stacked.stack(_models(cifar10.network, 2)).channels_interleaved
    assert not stacked.stack(_models(imdb.network, 2)).channels_interleaved


@pytest.mark.parametrize("name", sorted(NETWORKS))
def test_stack_unstack_round_trip_is_bit_identical(name):
    network, _ = NETWORKS[name]
    models = _models(network, 3)
    before = [{k: v.clone() for k, v in model.state_dict().items()} for model in models]
    net = stacked.stack(models)
    for pname, p in net.named_parameters():
        assert p.shape[0] == 3
        for k, model in enumerate(models):
            assert torch.equal(p[k], model.get_parameter(pname))
    with torch.no_grad():                      # scribble over the originals, then write the stack back
        for model in models:
            for p in model.parameters():
                p.fill_(7.0)
    assert net.unstack() is net.sources
    for model, want in zip(models, before):
        got = model.state_dict()
        assert list(got) == list(want)
        assert all(torch.equal(got[k], want[k]) for k in want)


def test_mismatched_architectures_raise_value_error():
    with pytest.raises(ValueError):
        stacked.stack([mnist.network(), cifar10.network()])
    narrow = KerasSequential(*list(mnist.network().children())[:-1], Dense(5 * 5 * 64, 9, "softmax"))
    with pytest.raises(ValueError, match="shape"):
        stacked.stack([mnist.network(), narrow])
    other_rate = mnist.network()
    other_rate[5].p = 0.25
    with pytest.raises(ValueError):
        stacked.stack([mnist.network(), other_rate])
    with pytest.raises(ValueError):
        stacked.stack([])
    with pytest.raises(ValueError):
        stacked.stack([mnist.network()] * 2, seeds=[1])


def test_an_unknown_child_raises_type_error_naming_it():
    class Squash(torch.nn.Module):
        def forward(self, x):
            return torch.tanh(x)

    net = KerasSequential(Dense(4, 4), Squash(), Dense(4, 2, "softmax"))
    with pytest.raises(TypeError, match="Squash"):
        stacked.stack([net])
    with pytest.raises(TypeError, match="Sequential"):
        stacked.stack([torch.nn.Sequential(torch.nn.Linear(2, 2))])


@pytest.mark.parametrize("name", ["mnist", "cifar10", "imdb"])
def test_seeds_give_keras_initialize_of_the_same_seed(name):
    network, _ = NETWORKS[name]
    seeds = [5, 17, 5]
    net = stacked.stack(_models(network, 3, seed=1), seeds=seeds)
    for k, seed in enumerate(seeds):
        want = keras_initialize(network(), torch.Generator().manual_seed(seed))
        for pname, p in want.named_parameters():
            assert torch.equal(net.get_parameter(pname)[k], p), (k, pname)
    first = next(net.parameters())
    assert torch.equal(first[0], first[2]) and not torch.equal(first[0], first[1])
