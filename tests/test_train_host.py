"""The training kernels' argument checks without a GPU: the wrappers of engine.py refuse before any launch, and the
C ABI's checks of tip_keras_adam, tip_softmax_xent_seg and tip_stack_gather return an error on host buffers (a
refused call never launches, so no device is touched)."""
import ctypes as C

import numpy as np
import pytest
import torch

import simple_tip_b200
from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E


@pytest.fixture
def no_launch(monkeypatch):
    """A wrapper that misses a check reaches _lib.load() and fails here instead of launching; the launch counter
    stays where it was."""
    before = _lib.launch_count()

    def refuse():
        raise AssertionError("the wrapper reached the library")

    monkeypatch.setattr(simple_tip_b200._lib, "load", refuse)
    yield
    monkeypatch.undo()
    assert _lib.launch_count() == before


def _xent_args(rows=4, classes=3):
    return (torch.zeros(rows, classes), torch.zeros(rows, classes), torch.zeros(1), torch.zeros(rows, classes),
            torch.zeros(1, dtype=torch.int32))


@pytest.mark.parametrize("which, bad", [("loss", torch.zeros(1, dtype=torch.float64)), ("loss", torch.zeros(0)),
                                        ("correct", torch.zeros(1, dtype=torch.int64)),
                                        ("correct", torch.zeros(0, dtype=torch.int32))])
def test_softmax_xent_refuses_a_bad_loss_or_correct(no_launch, which, bad):
    z, y, loss, dz, correct = _xent_args()
    args = {"loss": loss, "correct": correct, which: bad}
    with pytest.raises(ValueError, match=r"loss \(float32\) and correct \(int32\) need 1 elements"):
        E.softmax_xent(z, y, args["loss"], dz, args["correct"])


def test_softmax_xent_seg_refuses_a_bad_loss_or_correct(no_launch):
    z, y = torch.zeros(3, 4, 2), torch.zeros(3, 4, 2)
    with pytest.raises(ValueError, match="need 3 elements"):
        E.softmax_xent_seg(z, y, torch.zeros(2), None, torch.zeros(3, dtype=torch.int32))
    with pytest.raises(ValueError, match="need 3 elements"):
        E.softmax_xent_seg(z, y, torch.zeros(3), None, torch.zeros(3))


def test_the_xent_wrappers_refuse_host_tensors(no_launch):
    z, y, loss, dz, correct = _xent_args()
    for d in (dz, None):
        with pytest.raises(ValueError, match="one CUDA device"):
            E.softmax_xent(z, y, loss, d, correct)
    with pytest.raises(ValueError, match="one CUDA device"):
        E.softmax_xent_seg(z[None], y[None], loss, dz[None], correct)


def test_stack_gather_refuses_host_pools(no_launch):
    rows = torch.zeros(2, 4, dtype=torch.int64)
    perm = torch.arange(4).expand(2, 4).contiguous()
    with pytest.raises(ValueError, match="CUDA"):
        E.stack_gather(torch.zeros(10, 3), rows, perm, 0, 4, check=False)


def _lib_error():
    return _lib.load().tip_last_error().decode()


def _adam(n_tensors):
    table = (_lib.AdamTensor * 257)()
    state = np.zeros(2, np.int32)
    return _lib.load().tip_keras_adam(C.cast(table, C.c_void_p), n_tensors, 0, state.ctypes.data, 1e-3, 0.9, 0.999,
                                      1e-7, None)


@pytest.mark.parametrize("n_tensors", [0, 257, -1])
def test_c_abi_keras_adam_takes_1_to_256_tensors(n_tensors):
    before = _lib.launch_count()
    assert _adam(n_tensors) != 0
    assert "1..256 tensors per table" in _lib_error()
    assert _lib.launch_count() == before


def _xent_seg(segments=2, rows=3, classes=4):
    buf = np.zeros(64, np.float32)
    out = np.zeros(8, np.int32)
    return _lib.load().tip_softmax_xent_seg(buf.ctypes.data, buf.ctypes.data, segments, rows, classes,
                                            buf.ctypes.data, None, out.ctypes.data, None)


@pytest.mark.parametrize("args, msg", [(dict(segments=0), "1..2^31-1 segments"),
                                       (dict(segments=2 ** 31), "1..2^31-1 segments"),
                                       (dict(rows=0), "at least one row per segment"),
                                       (dict(classes=0), "1..32 classes"), (dict(classes=33), "1..32 classes")])
def test_c_abi_softmax_xent_seg_checks(args, msg):
    before = _lib.launch_count()
    assert _xent_seg(**args) != 0
    assert msg in _lib_error()
    assert _lib.launch_count() == before


def test_c_abi_softmax_xent_checks_its_classes():
    buf = np.zeros(64, np.float32)
    out = np.zeros(1, np.int32)
    assert _lib.load().tip_softmax_xent(buf.ctypes.data, buf.ctypes.data, 4, 33, buf.ctypes.data, None,
                                        out.ctypes.data, None) != 0
    assert "1..32 classes" in _lib_error()


def _gather(dtype=_lib.TIP_F32, row_elems=6, n_rows=5, n_perm=4, start=0, b=4, models=2, channels=0):
    pool = np.zeros(64, np.float64)
    idx = np.zeros(16, np.int64)
    return _lib.load().tip_stack_gather(pool.ctypes.data, dtype, row_elems, idx.ctypes.data, n_rows, idx.ctypes.data,
                                        n_perm, start, b, models, channels, pool.ctypes.data, None)


@pytest.mark.parametrize("args, msg", [
    (dict(dtype=_lib.TIP_BF16), "float32, float64 or int32 pool"),
    (dict(dtype=_lib.TIP_I16), "float32, float64 or int32 pool"),
    (dict(start=1), "batch [start, start + b) within the permutation"),
    (dict(start=-1, b=1), "batch [start, start + b) within the permutation"),
    (dict(n_perm=6), "perm indexes the first n_perm of each model's n_rows rows"),
    (dict(channels=4), "row_elems is pixels x channels"),
    (dict(channels=-3), "row_elems is pixels x channels"),
    (dict(row_elems=0), "empty rows or batch"),
])
def test_c_abi_stack_gather_checks(args, msg):
    before = _lib.launch_count()
    assert _gather(**args) != 0
    assert msg in _lib_error()
    assert _lib.launch_count() == before


def test_abi_signatures():
    lib = _lib.load()
    assert list(lib.tip_keras_adam.argtypes) == [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p] + [C.c_float] * 4 + \
        [C.c_void_p]
    assert list(lib.tip_softmax_xent_seg.argtypes) == [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32] + \
        [C.c_void_p] * 4
    assert list(lib.tip_stack_gather.argtypes) == [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                                   C.c_void_p] + [C.c_int64] * 5 + [C.c_void_p] * 2
