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

`fit_stack(models, x, y, rows, ...)` trains M models of one architecture together, each on its own rows of one
pool, with `fit`'s behaviour per model: one stacked network (`case_studies.stacked`), one `tip_stack_gather` per
tensor and one graph replay per step for all M.
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
    eagerly (the same operations, for comparison).  `load(perm, start)` fills the static batch with rows
    perm[start:start + B] of the training set."""

    def __init__(self, model, opt: KerasAdam, x, y, b: int, stats, graph: bool, pool=None):
        self.x, self.y = x, y
        self._capture(model, opt, x[:b].clone(), y[:b].clone(), b, 1, stats, graph, pool)

    def _capture(self, model, opt, xb, yb, b, segments, stats, graph, pool):
        import torch

        self.model, self.opt, self.xb, self.yb, self.b = model, opt, xb, yb, b
        dev = yb.device
        self.loss = torch.zeros(segments, dtype=torch.float32, device=dev)
        self.correct = torch.zeros(segments, dtype=torch.int32, device=dev)
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

    def _head(self, z):
        E.softmax_xent(z, self.yb, self.loss, self.dz, self.correct)

    def _grads(self):
        import torch

        z = self.model.logits(self.xb)
        self._head(z)
        # cuDNN hands a convolution's weight gradient over in the channels_last layout of its input; Adam's table
        # pairs elements by offset, so every gradient is laid out as its (contiguous) parameter
        return [g.contiguous() for g in torch.autograd.grad(z, self.opt.params, self.dz)]

    def _body(self, eager: bool = False):
        grads = self._grads()
        self.opt.step(self.opt.table(grads) if eager else self.table)
        self.loss_sum += self.loss.double() * self.b
        self.correct_sum += self.correct
        return grads

    def load(self, perm, start: int):
        import torch

        idx = perm[start:start + self.b]
        torch.index_select(self.x, 0, idx, out=self.xb)
        torch.index_select(self.y, 0, idx, out=self.yb)

    def __call__(self, perm, start: int):
        self.load(perm, start)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._body(eager=True)


class _StackStep(_Step):
    """One step of a stack of M models (`fit_stack`): the batch of every model gathered by `tip_stack_gather` (into
    the stack's input layout and [M, B, C] targets), the loss head `tip_softmax_xent_seg` with one segment per
    model, so each model's gradient is that of its own batch mean."""

    def __init__(self, net, opt: KerasAdam, x, y, rows, b: int, stats, graph: bool, pool=None):
        import torch

        self.x, self.y, self.rows, self.interleaved = x, y, rows, net.channels_interleaved
        m, dev = rows.shape[0], y.device
        first = torch.zeros((m, b), dtype=torch.int64, device=dev)        # any rows will do before the first load
        xb = E.stack_gather(x, rows, first, 0, b, self.interleaved, check=False)
        yb = E.stack_gather(y, rows, first, 0, b, check=False)
        self._capture(net, opt, xb, yb, b, m, stats, graph, pool)

    def _head(self, z):
        E.softmax_xent_seg(z, self.yb, self.loss, self.dz, self.correct)

    def load(self, perm, start: int):
        E.stack_gather(self.x, self.rows, perm, start, self.b, self.interleaved, out=self.xb, check=False)
        E.stack_gather(self.y, self.rows, perm, start, self.b, out=self.yb, check=False)


def _epochs(model, n: int, batch_size: int, epochs: int, draw, new_step, stats, validate, histories):
    """Keras' epoch loop, shared by `fit` (one model) and `fit_stack` (a stack of M): per epoch a fresh permutation
    `draw()`, its batches in order (the last one partial) through one step per batch size `new_step(b)`, then each
    model's mean loss and accuracy over the epoch from `stats` (float64 / int64 sums, one per model) and
    `validate()` = (val losses, val accuracies) per model or None, appended to `histories` (one per model)."""
    steps: Dict[int, _Step] = {}
    model.train()
    for epoch in range(epochs):
        perm = draw()
        for s in stats:
            s.zero_()
        for start in range(0, n, batch_size):
            b = min(batch_size, n - start)
            if b not in steps:
                steps[b] = new_step(b)
            steps[b](perm, start)
        val = validate()
        for k, (loss_sum, correct_sum) in enumerate(zip(stats[0].tolist(), stats[1].tolist())):
            history = histories[k]
            history["loss"].append(float(loss_sum) / n)
            history["accuracy"].append(int(correct_sum) / n)
            if val is not None:
                history["val_loss"].append(val[0][k])
                history["val_accuracy"].append(val[1][k])
        model.train()
        for history in histories:
            LOG.info("epoch %d/%d: %s", epoch + 1, epochs, {k: v[-1] for k, v in history.items() if v})
    model.eval()
    return histories


def _new_history() -> Dict[str, List[float]]:
    return {"loss": [], "accuracy": [], "val_loss": [], "val_accuracy": []}


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

    def validate():
        if not n_val:
            return None
        val_loss, val_acc = evaluate(model, x_val, y_val)
        return [val_loss], [val_acc]
    model.history = _epochs(model, n, batch_size, epochs, lambda: torch.randperm(n, device=dev, generator=shuffles),
                            lambda b: _Step(model, opt, x_tr, y_tr, b, stats, graph, pool), stats, validate,
                            [_new_history()])[0]
    return model


def fit_stack(models, x, y, rows, batch_size: int, epochs: int, validation_split: float = 0.1,
              seeds: Optional[List[int]] = None):
    """`fit` for M models of one architecture trained together in one stack (`case_studies.stacked`): model k's
    data set is `x[rows[k]], y[rows[k]]`, and for each model the behaviour is that of
    `fit(models[k], x[rows[k]], y[rows[k]], batch_size, epochs, validation_split)`: the last
    `validation_rows(n)` rows of rows[k] are held out and evaluated every epoch, every epoch walks a fresh
    permutation of the model's own training rows (independent between models) in batches, the last one partial, and
    the loss is the mean over the model's own batch rows, followed by Keras' Adam.  Returns the models, in eval
    mode, each with its own `history`.

    x, y: one pool on the models' CUDA device, y float32 one-hot [N, C]; x float32, float64 (used as float32, as
    the networks cast it) or int32 (token ids).  rows: int64 [M, n] on that device, checked once against the pool.
    seeds: None keeps the weights and draws the shuffles from torch's default CUDA generator; M ints start model k
    from the weights `fit(seed=seeds[k])` gives it (the same host generator draws), the shuffles coming from one
    device generator seeded with seeds[0].

    Each step is one `tip_stack_gather` per tensor (inputs, targets) plus one graph replay holding the stacked
    forward, `tip_softmax_xent_seg`, the backward and one `tip_keras_adam` over the stacked parameters (element-wise,
    so each model's update is its own Adam update).  A stack's shuffles and dropout draws are not those of M `fit`
    calls, and its grouped convolutions and batched GEMMs round differently: a model trained in a stack equals its
    single-model fit to rounding only (DESIGN.md §9)."""
    import torch

    from ..case_studies import stacked

    models = list(models)
    if not models:
        raise ValueError("fit_stack takes at least one model")
    if not (isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor) and isinstance(rows, torch.Tensor)
            and x.is_cuda and y.device == x.device and rows.device == x.device):
        raise ValueError("fit_stack takes x, y and rows as torch tensors on one CUDA device")
    if y.dim() != 2 or y.dtype != torch.float32 or y.shape[0] != x.shape[0]:
        raise ValueError(f"y must be float32 one-hot [{x.shape[0]}, C], got {tuple(y.shape)} {y.dtype}")
    if rows.dim() != 2 or rows.shape[0] != len(models):
        raise ValueError(f"rows must be [{len(models)}, n], got {tuple(rows.shape)}")
    if any(p.device != x.device for m in models for p in m.parameters()):
        raise ValueError("the models' parameters must live on the pool's device")
    m_count, n_all = rows.shape
    n_val = validation_rows(n_all, validation_split)
    n = n_all - n_val
    if n < 1:
        raise ValueError(f"no training rows left of {n_all} with validation_split={validation_split}")
    dev = x.device
    x, y, rows = x.contiguous(), y.contiguous(), rows.contiguous()
    E.check_stack_rows(rows, x.shape[0])
    net = stacked.stack(models, seeds)
    shuffles = None if seeds is None else torch.Generator(device=dev).manual_seed(int(seeds[0]))
    opt = KerasAdam(net.parameters())
    stats = (torch.zeros(m_count, dtype=torch.float64, device=dev),
             torch.zeros(m_count, dtype=torch.int64, device=dev))
    pool = torch.cuda.graph_pool_handle()
    perm = torch.empty((m_count, n), dtype=torch.int64, device=dev)

    def draw():
        for k in range(m_count):
            perm[k] = torch.randperm(n, device=dev, generator=shuffles)
        return perm
    val_rows = rows[:, n:].contiguous()

    def validate():
        if not n_val:
            return None
        return evaluate_stack(net, x, y, val_rows, max(batch_size, EVAL_ROWS // m_count))
    histories = _epochs(net, n, batch_size, epochs, draw,
                        lambda b: _StackStep(net, opt, x, y, rows, b, stats, True, pool), stats, validate,
                        [_new_history() for _ in models])
    net.unstack()
    for model, history in zip(models, histories):
        model.eval()
        model.history = history
    return models


def evaluate_stack(net, x, y, rows, batch: int):
    """([mean softmax cross-entropy], [accuracy]) per model of a stack in eval mode, model m on its rows
    `x[rows[m]]` against one-hot `y[rows[m]]` (rows int64 [M, n], checked by the caller; `tip_stack_gather` and
    `tip_softmax_xent_seg` per pass of `batch` rows per model; the loss is the exact row mean)."""
    import torch

    m, n = rows.shape
    dev = y.device
    order = torch.arange(n, dtype=torch.int64, device=dev).expand(m, n).contiguous()
    loss = torch.zeros(m, dtype=torch.float32, device=dev)
    correct = torch.zeros(m, dtype=torch.int32, device=dev)
    loss_sum = torch.zeros(m, dtype=torch.float64, device=dev)
    correct_sum = torch.zeros(m, dtype=torch.int64, device=dev)
    net.eval()
    with torch.no_grad():
        for start in range(0, n, batch):
            b = min(batch, n - start)
            xb = E.stack_gather(x, rows, order, start, b, net.channels_interleaved, check=False)
            yb = E.stack_gather(y, rows, order, start, b, check=False)
            E.softmax_xent_seg(net.logits(xb), yb, loss, None, correct)
            loss_sum += loss.double() * b
            correct_sum += correct
    return [v / n for v in loss_sum.tolist()], [v / n for v in correct_sum.tolist()]


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
