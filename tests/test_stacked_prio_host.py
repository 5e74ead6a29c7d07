"""Scoring the fault predictors of a model stack, host side without a GPU: tip_mc_head_stack's C ABI signature and
argument checks, the stacked head parser, the refusals of get_pred_and_uncertainty_stack, evaluate_stack and the
runner, and the stacked accuracies of active learning on the host."""
import ctypes as C

import numpy as np
import pytest
import torch

from simple_tip_b200 import _lib
from simple_tip_b200.case_studies import imdb, mnist
from simple_tip_b200.case_studies.stacked import stack
from simple_tip_b200.core import active_learning as AL
from simple_tip_b200.core import activations as A
from simple_tip_b200.core import prioritization as P


def test_abi_signature():
    fn = _lib.load().tip_mc_head_stack
    assert fn.restype == C.c_int
    assert list(fn.argtypes) == [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                 C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]


def _table(models, *layers):
    keep = [(np.zeros((models, i, o), np.float32), np.zeros((models, o), np.float32)) for i, o, _, _ in layers]
    table = (_lib.McLayer * len(layers))()
    for t, ((i, o, p, act), (k, b)) in enumerate(zip(layers, keep)):
        table[t] = _lib.McLayer(k.ctypes.data, b.ctypes.data, p, i, o, act, 0)
    return table, keep


def _call(layers, models=2, rows=0, ldm=None, seeds=True, samples=3, mode=_lib.MC_OUTPUT, ld=None):
    """rows = 0 (or models = 0) returns after the checks, so this runs without a device."""
    table, _keep = _table(max(models, 1), *layers)
    d = layers[0][0]
    h = np.zeros(max(models, 1) * d, np.float32)
    out = np.zeros(1, np.float32)
    seed_arr = (C.c_uint64 * max(models, 1))(*range(max(models, 1)))
    return _lib.load().tip_mc_head_stack(h.ctypes.data, models, rows, d if ld is None else ld,
                                         d if ldm is None else ldm, 0, 0, samples, table, len(layers),
                                         seed_arr if seeds else None, mode, out.ctypes.data, None)


@pytest.mark.parametrize("layers, ok", [
    ([(1600, 10, 0.5, _lib.MC_SOFTMAX)], True),
    ([(32, 20, 0.1, _lib.MC_RELU), (20, 2, 0.1, _lib.MC_SOFTMAX)], True),
    ([(8192, 64, 1.0, _lib.MC_LINEAR)] + [(64, 64, 0.0, _lib.MC_RELU)] * 3, True),
    ([(8193, 10, 0.5, _lib.MC_SOFTMAX)], False),
    ([(16, 65, 0.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 1.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 0.5, _lib.MC_SOFTMAX), (8, 2, 0.5, _lib.MC_LINEAR)], False),
    ([(16, 8, 0.5, _lib.MC_RELU), (9, 2, 0.5, _lib.MC_LINEAR)], False),
    ([(4, 4, 0.0, _lib.MC_RELU)] * 5, False),
])
def test_c_abi_checks_the_heads_as_tip_mc_head_does(layers, ok):
    rc = _call(layers)
    assert (rc == 0) == ok, _lib.load().tip_last_error()


def test_c_abi_checks_the_stack_arguments():
    head = [(16, 4, 0.5, _lib.MC_SOFTMAX)]
    assert _call(head) == 0
    assert _call(head, ldm=0) == 0                       # every model reads the same rows
    assert _call(head, models=0, seeds=False) == 0
    assert _call(head, seeds=False) != 0
    assert _call(head, models=-1) != 0
    assert _call(head, ldm=-1) != 0
    assert _call(head, ld=15) != 0
    assert _call(head, samples=0) != 0
    assert _call(head, mode=7) != 0


def test_stacked_head_parser():
    at, layers = A.mc_head_layers_stack(stack([mnist.network(), mnist.network()]))
    assert at == 5 and [(l.p, type(l.module).__name__, l.activation) for l in layers] == [(0.5, "StackedDense",
                                                                                           "softmax")]
    kernel, bias, p, act = A._head_tensors(layers, torch.device("cpu"))[0]
    assert kernel.shape == (2, 1600, 10) and bias.shape == (2, 10) and (p, act) == (0.5, "softmax")
    at, layers = A.mc_head_layers_stack(stack([imdb.network()] * 3))
    assert at == 4 and [(l.p, l.activation) for l in layers] == [(0.1, "relu"), (0.1, "softmax")]
    assert [tuple(l.module.kernel.shape) for l in layers] == [(3, 32, 20), (3, 20, 2)]
    with pytest.raises(ValueError, match="StackedSequential"):
        A.mc_head_layers_stack(mnist.network())


def test_stacked_scoring_refuses_before_any_work():
    net = stack([mnist.network(), mnist.network()])
    x = np.zeros((2, 28, 28, 1), np.float32)
    with pytest.raises(ValueError, match="StackedSequential"):
        A.get_pred_and_uncertainty_stack(mnist.network(), x)
    with pytest.raises(ValueError, match="seeds"):
        A.get_pred_and_uncertainty_stack(net, x, seeds=[0])
    with pytest.raises(ValueError, match="sampler"):
        A.get_pred_and_uncertainty_stack(net, x, sampler="tf")


def test_evaluate_stack_refuses_before_any_forward_pass():
    models = [mnist.network(), mnist.network()]
    x, y = np.zeros((3, 28, 28, 1), np.float32), np.zeros(3)
    args = dict(training_dataset=x, nominal_test_dataset=x, nominal_test_labels=y, ood_test_dataset=x,
                ood_test_labels=y, nc_activation_layers=[0], sa_activation_layers=[0])
    with pytest.raises(ValueError, match="model ids"):
        P.evaluate_stack([0], "mnist", models, **args)
    with pytest.raises(ValueError, match="repeat"):
        P.evaluate_stack([1, 1], "mnist", models, **args)
    with pytest.raises(ValueError, match="_"):
        P.evaluate_stack([0, 1], "mn_ist", models, **args)
    with pytest.raises(ValueError, match="labels"):
        P.evaluate_stack([0, 1], "mnist", models, **dict(args, ood_test_labels=np.zeros(4)))


def test_runner_refuses_an_empty_stack_size():
    datasets = ((np.zeros((4, 28, 28, 1), np.float32), np.zeros(4)),) * 3
    cs = mnist.MnistCaseStudy("unused", datasets, device="cpu")
    with pytest.raises(ValueError, match="stack_size"):
        cs.run_prio_eval([0, 1], stacked=True, stack_size=0)


def test_stacked_accuracies_on_the_host():
    torch.manual_seed(0)
    models = [mnist.network() for _ in range(4)]
    net = stack(models).eval()
    x = torch.rand(50, 28, 28, 1)
    y = torch.randint(0, 10, (50,))
    got = AL.accuracies_stack(net, x, y, batch_size=16)
    with torch.no_grad():
        probs = torch.cat([net(net.stack_inputs([x[s:s + 16]] * 4)) for s in range(0, 50, 16)], dim=1)
    assert got == [int((probs[m].argmax(dim=1) == y).sum()) / 50 for m in range(4)]


def test_modules_that_do_not_stack_are_evaluated_one_by_one():
    torch.manual_seed(1)
    plain = [torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(12, 3), torch.nn.Softmax(dim=1)) for _ in range(2)]
    x, y = torch.rand(20, 3, 4), torch.randint(0, 3, (20,))
    datasets = {("nominal", "observed"): (x, y), ("ood", "future"): (x[:7], y[:7])}
    got = AL._evaluate_stack(plain, datasets, 3, batch_size=8)
    assert got == [AL._evaluate(m, datasets, 3, batch_size=8) for m in plain]
