"""Keras' `Model.fit` for the case studies' torch models (case_study_*.py `_train_new_model`), with CUDA graphs.

`fit(model, x, y, batch_size, epochs, validation_split)` is what the case studies call after
`model.compile(loss="categorical_crossentropy", optimizer="adam", metrics=["accuracy"])`: the last
`len(x) - floor(len(x) * (1 - validation_split))` rows are held out and only evaluated, every epoch draws a fresh
permutation of the training rows on the device and walks it in batches (the last one partial), and each step is
forward, `tip_softmax_xent` (the loss head), backward and `tip_keras_adam` (Keras' Adam over every parameter in one
launch).  A step is captured once per batch shape as a CUDA graph; replaying it costs the device gather of the batch
into the graph's static inputs plus one graph launch.  Dropout stays random across replays: torch's CUDA generator
is registered with every graph it is captured in.

The model is a `torch.nn.Module` with a `logits(x)` method (the last Dense layer's input to its softmax) and float32
parameters, as the networks of `simple_tip_b200.case_studies` are.  Training moves nothing to the host but one
loss and one accuracy count per epoch.
"""
from __future__ import annotations

import ctypes
import logging
import math
from typing import Dict, List, Optional

import numpy as np

from .. import _lib
from .. import engine as E

LOG = logging.getLogger(__name__)

ADAM = dict(lr=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-7)      # tf.keras.optimizers.Adam() defaults (TF 2.6)
EVAL_ROWS = 1024        # rows per forward pass of the validation split


def validation_rows(n: int, validation_split: float) -> int:
    """Rows Keras holds out of n (`train_validation_split`: split_at = int(floor(n * (1 - validation_split))))."""
    return n - int(math.floor(n * (1.0 - validation_split)))


def keras_fans(shape) -> tuple:
    """(fan_in, fan_out) of a kernel of Keras shape `shape` (keras.initializers `_compute_fans`): the last two
    dimensions are (in, out), every leading one is a receptive field."""
    shape = tuple(int(s) for s in shape)
    if len(shape) < 1:
        return 1, 1
    if len(shape) == 1:
        return shape[0], shape[0]
    receptive = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    return shape[-2] * receptive, shape[-1] * receptive


def glorot_limit(shape) -> float:
    fan_in, fan_out = keras_fans(shape)
    return math.sqrt(6.0 / (fan_in + fan_out))


def uniform_(t, limit: float, generator=None):
    """t <- U(-limit, limit), drawn on the host from `generator` (None: torch's default generator)."""
    import torch

    with torch.no_grad():
        u = torch.rand(t.shape, generator=generator, dtype=torch.float32)
        t.copy_((u * 2.0 - 1.0) * limit)
    return t


def keras_initialize(model, generator=None):
    """Applies every submodule's Keras initialisers (`keras_init(generator)`: glorot_uniform kernels, zero biases,
    Embedding U(-0.05, 0.05), LayerNorm ones / zeros) in `model.modules()` order."""
    for m in model.modules():
        init = getattr(m, "keras_init", None)
        if init is not None:
            init(generator)
    return model


class KerasAdam:
    """Adam's moments and step counter for a list of float32 CUDA parameters (`tip_keras_adam`)."""

    def __init__(self, params, lr=ADAM["lr"], beta1=ADAM["beta1"], beta2=ADAM["beta2"], epsilon=ADAM["epsilon"]):
        import torch

        self.params = list(params)
        self.m = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self.v = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self.state = torch.zeros(2, dtype=torch.int32, device=self.params[0].device)
        self.numel = sum(p.numel() for p in self.params)
        self.hyper = (lr, beta1, beta2, epsilon)

    def table(self, grads, out=None):
        return E.adam_table([p.detach() for p in self.params], grads, self.m, self.v, out=out)

    def step(self, table):
        E.keras_adam(table, len(self.params), self.numel, self.state, *self.hyper)


class _Step:
    """One training step at batch size B on static device buffers, captured as a CUDA graph (graph=True) or run
    eagerly (the same operations, for comparison)."""

    def __init__(self, model, opt: KerasAdam, x, y, b: int, stats, graph: bool, pool=None):
        import torch

        self.model, self.opt, self.x, self.y, self.b = model, opt, x, y, b
        dev = y.device
        self.xb = x[:b].clone()
        self.yb = y[:b].clone()
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.correct = torch.zeros(1, dtype=torch.int32, device=dev)
        self.dz = torch.empty_like(self.yb)
        self.loss_sum, self.correct_sum = stats
        self.graph = None
        if graph:
            side = torch.cuda.Stream(dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):         # warm-up: library handles and algorithm choices, no update
                for _ in range(2):
                    self._grads()
            torch.cuda.current_stream(dev).wait_stream(side)
            self.table = torch.empty(len(opt.params) * ctypes.sizeof(_lib.AdamTensor), dtype=torch.uint8, device=dev)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, pool=pool):
                self.grads = self._body()
            opt.table(self.grads, out=self.table)

    def _grads(self):
        import torch

        z = self.model.logits(self.xb)
        E.softmax_xent(z, self.yb, self.loss, self.dz, self.correct)
        # cuDNN hands a convolution's weight gradient over in the channels_last layout of its input; Adam's table
        # pairs elements by offset, so every gradient is laid out as its (contiguous) parameter
        return [g.contiguous() for g in torch.autograd.grad(z, self.opt.params, self.dz)]

    def _body(self, eager: bool = False):
        grads = self._grads()
        self.opt.step(self.opt.table(grads) if eager else self.table)
        self.loss_sum += self.loss.double() * self.b
        self.correct_sum += self.correct
        return grads

    def __call__(self, idx):
        import torch

        torch.index_select(self.x, 0, idx, out=self.xb)
        torch.index_select(self.y, 0, idx, out=self.yb)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._body(eager=True)


def fit(model, x, y, batch_size: int, epochs: int, validation_split: float = 0.1, seed: Optional[int] = None):
    """Keras' `model.fit(x, y, batch_size, epochs, validation_split)` for a categorical-cross-entropy softmax model,
    graph-captured; returns the model, in eval mode, with `model.history` = {"loss", "accuracy", "val_loss",
    "val_accuracy"} per epoch (also logged at INFO).

    x, y: torch tensors on the model's CUDA device, y float32 one-hot [N, C] (what `active_learning._retrain` hands
    a training process).  seed: None draws the shuffles from torch's default CUDA generator and keeps the model's
    weights; an int re-initialises the weights with Keras' initialisers from a host generator seeded with it and
    draws the shuffles from a device generator seeded with it (the reference's models are unseeded; the seed is for
    reproducible runs).

    The optimizer is Keras' Adam with its defaults as `tip_keras_adam` computes it; agreement with TensorFlow is at
    the level of that formula, not of TensorFlow's bits (TensorFlow is not a dependency).  The loss is the softmax
    cross-entropy of the logits, not Keras' `-log(clip(p, 1e-7, 1 - 1e-7))` of the probabilities: the two differ
    only where a true-class probability is below 1e-7 (DESIGN.md §9)."""
    return _fit(model, x, y, batch_size, epochs, validation_split, seed, graph=True)


def _fit(model, x, y, batch_size, epochs, validation_split, seed, graph):
    import torch

    if not (isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor) and x.is_cuda and y.device == x.device):
        raise ValueError("fit takes x and y as torch tensors on one CUDA device")
    if y.dim() != 2 or y.dtype != torch.float32 or y.shape[0] != x.shape[0]:
        raise ValueError(f"y must be float32 one-hot [{x.shape[0]}, C], got {tuple(y.shape)} {y.dtype}")
    n_val = validation_rows(x.shape[0], validation_split)
    n = x.shape[0] - n_val
    if n < 1:
        raise ValueError(f"no training rows left of {x.shape[0]} with validation_split={validation_split}")
    dev = x.device
    x, y = x.contiguous(), y.contiguous()
    x_tr, y_tr, x_val, y_val = x[:n], y[:n], x[n:], y[n:]
    shuffles = None
    if seed is not None:
        keras_initialize(model, torch.Generator().manual_seed(seed))
        shuffles = torch.Generator(device=dev).manual_seed(seed)
    opt = KerasAdam(model.parameters())
    stats = (torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev))
    pool = torch.cuda.graph_pool_handle() if graph else None
    steps: Dict[int, _Step] = {}
    history: Dict[str, List[float]] = {"loss": [], "accuracy": [], "val_loss": [], "val_accuracy": []}
    model.train()
    for epoch in range(epochs):
        perm = torch.randperm(n, device=dev, generator=shuffles)
        for s in stats:
            s.zero_()
        for start in range(0, n, batch_size):
            b = min(batch_size, n - start)
            if b not in steps:
                steps[b] = _Step(model, opt, x_tr, y_tr, b, stats, graph, pool)
            steps[b](perm[start:start + b])
        history["loss"].append(float(stats[0].item()) / n)
        history["accuracy"].append(int(stats[1].item()) / n)
        if n_val:
            val_loss, val_acc = evaluate(model, x_val, y_val)
            history["val_loss"].append(val_loss)
            history["val_accuracy"].append(val_acc)
        model.train()
        LOG.info("epoch %d/%d: %s", epoch + 1, epochs, {k: v[-1] for k, v in history.items() if v})
    model.eval()
    model.history = history
    return model


def evaluate(model, x, y, rows: int = EVAL_ROWS):
    """(mean softmax cross-entropy, accuracy) of the model in eval mode on x against one-hot y (`tip_softmax_xent`
    per pass of `rows` rows; the loss is the exact row mean)."""
    import torch

    dev = y.device
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    correct = torch.zeros(1, dtype=torch.int32, device=dev)
    loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
    correct_sum = torch.zeros(1, dtype=torch.int64, device=dev)
    model.eval()
    with torch.no_grad():
        for start in range(0, x.shape[0], rows):
            z = model.logits(x[start:start + rows]).contiguous()
            E.softmax_xent(z, y[start:start + rows].contiguous(), loss, None, correct)
            loss_sum += loss.double() * z.shape[0]
            correct_sum += correct
    return float(loss_sum.item()) / x.shape[0], int(correct_sum.item()) / x.shape[0]
