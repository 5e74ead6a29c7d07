"""The coverage arm of a model stack, host side without a GPU: tip_cam_bits_stack's C ABI signature against the header
and its argument checks, `StackedSequential.model_major` against `stack_inputs` and each model's own layers, and the
refusals of the stacked coverage worker, evaluate_stack and the runner before any forward pass."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from simple_tip_b200 import _lib
from simple_tip_b200.case_studies import cifar10, imdb, mnist, stacked
from simple_tip_b200.core import activations as A
from simple_tip_b200.core import coverage_worker as CW
from simple_tip_b200.core import prioritization as P

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200tip.h")
CTYPE = {"int64_t": C.c_int64, "int32_t": C.c_int32, "int": C.c_int}


def test_abi_signature_matches_the_header():
    decl = re.search(r"int tip_cam_bits_stack\(([^)]*)\);", open(HEADER).read()).group(1)
    want = []
    for arg in decl.split(","):
        kind = arg.strip().rsplit(" ", 1)[0]
        want.append(C.c_void_p if "*" in arg else CTYPE[kind])
    fn = _lib.load().tip_cam_bits_stack
    assert fn.restype == C.c_int
    assert list(fn.argtypes) == want
    assert len(want) == 12


def _call(models=3, n=5, words=2, max_rounds=2, null=None):
    """Host buffers stand in for device ones: every call here is refused before any launch."""
    bufs = {k: np.zeros(max(models * n * max(words, 1) * 2, 16), np.int32)
            for k in ("bits", "gain", "covered2", "cand", "order", "state")}
    ptr = {k: (None if k == null else v.ctypes.data) for k, v in bufs.items()}
    return _lib.load().tip_cam_bits_stack(ptr["bits"], models, n, words, ptr["gain"], ptr["covered2"], ptr["cand"],
                                          ptr["order"], ptr["state"], max_rounds, 1, None)


@pytest.mark.parametrize("null", ["bits", "gain", "covered2", "cand", "order", "state"])
def test_c_abi_refuses_null_pointers(null):
    assert _call(null=null) != 0
    assert "null pointer" in _lib.load().tip_last_error().decode()


@pytest.mark.parametrize("kw", [dict(models=0), dict(models=-1), dict(n=0), dict(n=-3), dict(words=0),
                                dict(max_rounds=-1), dict(models=2 ** 16, n=2 ** 15)])
def test_c_abi_refuses_bad_shapes(kw):
    assert _call(**kw) != 0
    assert "shape" in _lib.load().tip_last_error().decode()


# ---- the layout of a stack's hooked children ------------------------------------------------------------------------------
def _models(module, m, seed=0):
    torch.manual_seed(seed)
    return [module.network().eval() for _ in range(m)]


def _inputs(name, n, seed):
    g = torch.Generator().manual_seed(seed)
    if name == "imdb":
        return torch.randint(0, 2000, (n, 100), generator=g, dtype=torch.int32)
    if name == "cifar10":
        return torch.rand((n, 32, 32, 3), generator=g, dtype=torch.float64)
    return torch.rand((n, 28, 28, 1), generator=g)


NETS = {"mnist": mnist, "cifar10": cifar10, "imdb": imdb}


@pytest.mark.parametrize("name", sorted(NETS))
def test_model_major_inverts_stack_inputs_for_every_child(name):
    models = _models(NETS[name], 3)
    net = stacked.stack(models).eval()
    assert net.channels_interleaved == (name != "imdb")
    children = list(range(len(list(net.children())) - 1))
    acts = A.TransparentModel(net, children, include_last_layer=False).get_activations(
        net.stack_inputs([_inputs(name, 5, 1)] * 3))
    flatten_at = next((i for i, c in enumerate(net.children()) if isinstance(c, stacked.StackedFlatten)), None)
    for child, y in zip(children, acts):
        mm = net.model_major(child, y)
        assert mm.shape[:2] == (3, 5), (child, tuple(mm.shape))
        if net.channels_interleaved and child < flatten_at:         # the stack's input layout: [B, H, W, M * C]
            assert torch.equal(net.stack_inputs(list(mm)), y), child
        else:
            assert mm is y, child
    with pytest.raises(IndexError):
        net.model_major(len(children) + 1, acts[0])


@pytest.mark.parametrize("name", sorted(NETS))
def test_model_major_outputs_match_each_models_own_layers(name):
    module = NETS[name]
    models = _models(module, 3, seed=4)
    net = stacked.stack(models).eval()
    x = _inputs(name, 6, 2)
    layers = module.NC_ACTIVATION_LAYERS
    acts = A.TransparentModel(net, layers, include_last_layer=False).get_activations(net.stack_inputs([x] * 3))
    for m, model in enumerate(models):
        own = A.TransparentModel(model, layers, include_last_layer=False).get_activations(x)
        for child, y, want in zip(layers, acts, own):
            got = net.model_major(child, y)[m]
            assert got.shape == want.shape, (m, child)
            torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5 * float(want.abs().max()) + 1e-30)


# ---- refusals before any forward pass -------------------------------------------------------------------------------------
def _no_forward(net):
    def hook(*_):
        raise AssertionError("a forward pass ran before the refusal")
    for child in net.children():
        child.register_forward_pre_hook(hook)
    return net


def test_worker_refuses_before_any_forward_pass():
    net = _no_forward(stacked.stack(_models(mnist, 2)))
    x = np.zeros((4, 28, 28, 1), np.float32)
    with pytest.raises(ValueError, match="child indices"):
        CW.StackedCoverageWorker(net, [0, "1"], x)
    with pytest.raises(ValueError, match="child indices"):
        CW.StackedCoverageWorker(net, [True], x)
    with pytest.raises(ValueError, match="StackedSequential"):
        CW.StackedCoverageWorker(_no_forward(mnist.network()), [0], x)
    with pytest.raises(IndexError):
        CW.StackedCoverageWorker(net, [0, 9], x)
    with pytest.raises(ValueError, match="no inputs"):
        CW.StackedCoverageWorker(net, [0], x[:0])


def test_evaluate_stack_refuses_dotted_coverage_layers_before_any_forward_pass(monkeypatch):
    def no_stack(*_a, **_k):
        raise AssertionError("the stack was built before the refusal")
    monkeypatch.setattr(stacked, "stack", no_stack)
    models = _models(imdb, 2)
    x, y = np.zeros((3, 100), np.int32), np.zeros(3)
    args = dict(training_dataset=x, nominal_test_dataset=x, nominal_test_labels=y, ood_test_dataset=x,
                ood_test_labels=y, nc_activation_layers=[3, "2.ffn"], sa_activation_layers=[5])
    with pytest.raises(ValueError, match="child indices"):
        P.evaluate_stack([0, 1], "imdb", models, stacked_coverage=True, **args)


def test_runner_refuses_stacked_coverage_without_a_stack():
    datasets = ((np.zeros((4, 28, 28, 1), np.float32), np.zeros(4)),) * 3
    cs = mnist.MnistCaseStudy("unused", datasets, device="cpu")
    cs.load_model = lambda _i: pytest.fail("a model was loaded before the refusal")
    with pytest.raises(ValueError, match="stacked=True"):
        cs.run_prio_eval([0, 1], stacked_coverage=True)
