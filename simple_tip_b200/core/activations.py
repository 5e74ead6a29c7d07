"""Activation-trace producer for PyTorch models and the reference's on-disk badge layout
(SURVEY.md §8 f4).

The reference obtains activation traces from a multi-output Keras model
(`handler_model.BaseModel.get_activations / walk_activations`, handler_model.py:175-206) as host
NumPy arrays and can persist them in badges of 100 inputs
(`activation_persistor.py:13-35`: `<root>/activations/<case_study>/model_<id>/<dataset>/layer_<i>/badge_<b>.npy`,
labels in `.../labels/badge_<b>.npy`).  Here the same two things for a `torch.nn.Module`:

* `TransparentModel` returns the outputs of selected layers for a batch through forward hooks.  The
  tensors stay on the model's device: handed to `DSA` / `LSA` / `KMNC.buckets` / `DeepGini.calculate`
  they are scored without a host round trip (those entry points accept CUDA tensors).
* `persist_badges` / `load_badges` write and read the reference's `.npy` layout, so traces produced
  here can be consumed by the reference's scripts and vice versa.
"""
from __future__ import annotations

import os
from typing import Dict, Generator, Iterable, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np

BADGE_SIZE = 100      # activation_persistor.py:11

LayerId = Union[int, str]


class TransparentModel:
    """Selected layer outputs of a torch module, like the reference's transparent Keras model
    (handler_model.py:193-206: the outputs of `model.layers[i]` for i in `activation_layers`,
    plus the model output when `include_last_layer`).

    activation_layers: indices into `list(model.children())` (what Keras' `model.layers` is for a
    Sequential) or dotted submodule names from `model.named_modules()`."""

    def __init__(self, model, activation_layers: Optional[Sequence[LayerId]], include_last_layer: bool = True):
        if activation_layers is None:
            raise ValueError("No activation layers specified")          # handler_model.py:196-197
        self.model = model
        self.include_last_layer = include_last_layer
        children = list(model.children())
        named = dict(model.named_modules())
        self._modules = []
        for lid in activation_layers:
            if isinstance(lid, (int, np.integer)):
                if not 0 <= int(lid) < len(children):
                    raise IndexError(f"layer index {lid} out of range (model has {len(children)} layers)")
                self._modules.append(children[int(lid)])
            else:
                if lid not in named:
                    raise KeyError(f"no submodule named {lid!r}")
                self._modules.append(named[lid])

    def get_activations(self, x) -> List["torch.Tensor"]:     # noqa: F821
        """One deterministic forward pass (eval mode, no grad); returns one tensor per selected layer
        (+ the model output), each [batch, ...], on the model's device."""
        import torch

        captured: Dict[int, torch.Tensor] = {}
        hooks = [m.register_forward_hook(lambda _m, _i, out, k=k: captured.__setitem__(k, out.detach()))
                 for k, m in enumerate(self._modules)]
        was_training = self.model.training
        self.model.eval()
        try:
            with torch.no_grad():
                out = self.model(x)
        finally:
            for h in hooks:
                h.remove()
            self.model.train(was_training)
        missing = [k for k in range(len(self._modules)) if k not in captured]
        if missing:
            raise RuntimeError(f"selected layers {missing} did not run in the forward pass")
        acts = [captured[k] for k in range(len(self._modules))]
        if self.include_last_layer:
            acts.append(out.detach())
        return acts

    def walk_activations(self, batches: Iterable) -> Generator[List["torch.Tensor"], None, None]:   # noqa: F821
        """Activations badge by badge for a (potentially large) dataset (handler_model.py:175-180)."""
        for badge in batches:
            yield self.get_activations(badge)

    def collect(self, x, batch_size: int = BADGE_SIZE) -> List["torch.Tensor"]:   # noqa: F821
        """All of x in badges of `batch_size`; per layer one [N, ...] tensor on the model's device."""
        import torch

        per_layer: Optional[List[List[torch.Tensor]]] = None
        for start in range(0, x.shape[0], batch_size):
            acts = self.get_activations(x[start:start + batch_size])
            if per_layer is None:
                per_layer = [[] for _ in acts]
            for lst, a in zip(per_layer, acts):
                lst.append(a)
        if per_layer is None:
            return []
        return [torch.cat(lst, dim=0) for lst in per_layer]


class HookedModelHandler:
    """What the study's arms for a torch model share (`SurpriseHandler`, `CoverageWorker`): the hooked model in
    `self.base_model` (a `TransparentModel`), the device it runs on, and timers that include the device work."""

    base_model: TransparentModel

    def _model_device(self):
        import torch

        return next(iter(self.base_model.model.parameters()), torch.empty(0)).device

    def _inputs(self, data, what: str):
        """data as a tensor on the model's device; ValueError for an empty set"""
        import torch

        x = data if isinstance(data, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(data))
        if x.shape[0] == 0:
            raise ValueError(f"{what} holds no inputs")
        return x.to(self._model_device())

    def _synced(self, fn, timer):
        """fn() timed by `timer`, which stops after a synchronise of the current CUDA device (the scoring device)
        and of the model's device when that is another CUDA device."""
        from .. import engine as E

        return _synced(fn, timer, E.require_cuda(), self._model_device())


DROPOUT_SAMPLE_SIZE = 200      # handler_model.py:7
MC_ROWS_PER_PASS = 8192        # rows of one MC-dropout forward pass: a batch is replicated up to this many
MC_SAMPLERS = ("torch", "head")


class HeadLayer(NamedTuple):
    """One dense layer of an MC-dropout head: the dropout rate on its input (0: none), the module(s) it came from,
    and its activation (None, "relu" or "softmax")."""
    p: float
    module: object
    activation: Optional[str]


def mc_head_layers(model) -> Tuple[int, List[HeadLayer]]:
    """The model's MC-dropout head as `sampler="head"` samples it: (index of the first top-level dropout child, the
    dense layers from there on).  Like uncertainty-wizard's `stochastic_from_keras`, only the top-level dropout
    layers are stochastic; dropouts nested inside earlier children stay in eval mode.

    The model must be a `torch.nn.Sequential`; from its first `_DropoutNd` child on, every child must be a
    `torch.nn.Dropout`, a case-study `Dense` (activation None, "relu" or "softmax"), or a `torch.nn.Linear`
    optionally followed by `ReLU` or `Softmax(dim=-1 or 1)`; at most one dropout precedes a dense layer, the head
    ends in a dense layer, and a softmax ends it.  Anything else raises ValueError naming the module.  (-1, []) when
    the model has no dropout module at all."""
    import torch

    from ..case_studies.base import Dense

    if not isinstance(model, torch.nn.Sequential):
        raise ValueError(f"sampler='head' needs a torch.nn.Sequential model, got {type(model).__name__}")
    return _head_layers(model, Dense)


def mc_head_layers_stack(stack) -> Tuple[int, List[HeadLayer]]:
    """`mc_head_layers` for a `StackedSequential`: the same checks and messages, with `StackedDense` layers (kernel
    [M, in, out], bias [M, out]) in the place of Dense."""
    from ..case_studies.stacked import StackedDense, StackedSequential

    if not isinstance(stack, StackedSequential):
        raise ValueError(f"the stacked head sampler needs a StackedSequential, got {type(stack).__name__}")
    return _head_layers(stack, StackedDense)


def _head_layers(model, dense) -> Tuple[int, List[HeadLayer]]:
    """mc_head_layers' parse of a Sequential whose dense layers are `dense` modules."""
    import torch
    from torch.nn.modules.dropout import _DropoutNd

    children = list(model.children())
    first = next((i for i, m in enumerate(children) if isinstance(m, _DropoutNd)), -1)
    if first < 0:
        if any(isinstance(m, _DropoutNd) for m in model.modules()):
            raise ValueError("sampler='head' samples top-level dropout layers; this model's dropouts are all nested")
        return -1, []
    layers: List[HeadLayer] = []
    p = None
    i = first
    while i < len(children):
        m = children[i]
        where = f"child {i} ({type(m).__name__})"
        if layers and layers[-1].activation == "softmax":
            raise ValueError(f"sampler='head': {where} follows the head's softmax")
        if type(m) is torch.nn.Dropout:
            if p is not None:
                raise ValueError(f"sampler='head': {where} is a second dropout before one dense layer")
            p = float(m.p)
        elif isinstance(m, dense):
            if m.activation not in (None, "relu", "softmax"):
                raise ValueError(f"sampler='head': {where} has activation {m.activation!r}")
            layers.append(HeadLayer(p or 0.0, m, m.activation))
            p = None
        elif type(m) is torch.nn.Linear:
            act, nxt = None, children[i + 1] if i + 1 < len(children) else None
            if type(nxt) is torch.nn.ReLU:
                act = "relu"
            elif type(nxt) is torch.nn.Softmax and nxt.dim in (-1, 1):
                act = "softmax"
            layers.append(HeadLayer(p or 0.0, m, act))
            p = None
            i += act is not None
        else:
            raise ValueError(f"sampler='head' cannot sample {where}: the head after the first top-level dropout may "
                             "hold only Dropout, Dense and Linear (+ ReLU / Softmax) layers")
        i += 1
    if p is not None or not layers:
        raise ValueError("sampler='head': the head must end in a dense layer")
    if len(layers) > 4:
        raise ValueError(f"sampler='head' samples heads of at most 4 dense layers, this one has {len(layers)}")
    return first, layers


def _head_tensors(layers: Sequence[HeadLayer], dev):
    """(kernel [in, out], bias [out], p, activation) per layer as contiguous float32 on dev; Linear weights are
    transposed once.  A stack's StackedDense layers give kernel [M, in, out] and bias [M, out]."""
    import torch

    out = []
    for layer in layers:
        m = layer.module
        if isinstance(m, torch.nn.Linear):
            kernel = m.weight.detach().t()
            bias = m.bias.detach() if m.bias is not None else torch.zeros(m.out_features, device=m.weight.device)
        else:
            kernel, bias = m.kernel.detach(), m.bias.detach()
        out.append((kernel.to(dev, torch.float32).contiguous(), bias.to(dev, torch.float32).contiguous(), layer.p,
                    layer.activation))
    return out


def head_input(trunk: Sequence, n: int, models: Optional[int] = None):
    """The head's input captured batch by batch in the point pass, as one [n, D] tensor; ValueError unless every
    batch is 2-D float32 (a head of dense layers takes flat rows) and they hold n rows together.  With `models`, every
    batch is a stack's [models, B, D] chunk and the result is [models, n, D]."""
    import torch

    dims, want = (2, "2-D float32 [N, D]") if models is None else (3, f"3-D float32 [{models}, B, D]")
    for t in trunk:
        if t.dim() != dims or t.dtype != torch.float32 or (models is not None and t.shape[0] != models):
            raise ValueError(f"sampler='head' needs the head's input as {want}, got {tuple(t.shape)} {t.dtype}")
    rows = dims - 2
    h = torch.cat(list(trunk), dim=rows) if len(trunk) != 1 else trunk[0]
    if h.shape[rows] != n:
        raise ValueError(f"the head saw {h.shape[rows]} rows, the model's output has {n}")
    return h


def _synced(fn, timer, score_dev, model_dev):
    """fn() timed by `timer`, which stops after a synchronise of the scoring device and of the model's device when
    that is another CUDA device."""
    import torch

    with timer:
        res = fn()
        torch.cuda.synchronize(score_dev)
        if model_dev.type == "cuda" and model_dev != score_dev:
            torch.cuda.synchronize(model_dev)
    return res


def get_pred_and_uncertainty(model, x, batch_size: int = 32, sample_size: int = DROPOUT_SAMPLE_SIZE, seed: int = 0,
                             sampler: Optional[str] = None
                             ) -> Tuple[np.ndarray, Dict[str, np.ndarray], Dict[str, List[float]]]:
    """Point predictions and uncertainties of a torch model (handler_model.py:102-173, `BaseModel.get_pred_and_uncertainty`).

    The model's output is taken to be its softmax output, as in the study, whose models end in a softmax layer; wrap
    a model that returns logits (e.g. `torch.nn.Sequential(model, torch.nn.Softmax(dim=1))`) before calling this.

    Returns (pred, uncertainties, times) like the reference: pred is the argmax of the point pass (int64);
    uncertainties holds "softmax", "pcs", "softmax_entropy" and "deep_gini" as stored by the study
    (`as_confidence=False`: the max softmax and PCS are negated) and, when the model has dropout modules, "VR", the
    variation ratio over `sample_size` MC-dropout samples; times[name] = [0, prediction time, quantifier time, 0]
    in seconds.  `x` must hold at least one input (ValueError otherwise).

    The model runs wherever its parameters live (the host, or any CUDA device); `x` is moved there.  Its outputs
    are scored on the current CUDA device: they are copied there when the model lives elsewhere.

    The point pass runs in eval mode without gradients.  The MC-dropout passes switch only the dropout modules
    (`torch.nn.modules.dropout._DropoutNd`) to training mode — batch norm and everything else stays in eval mode —
    and restore every module's mode afterwards.  Each batch of `batch_size` inputs is replicated along the batch
    dimension up to MC_ROWS_PER_PASS rows per forward pass; every pass's votes go straight to `tip_vote_add`, so
    the [N, sample_size, C] samples are never held at once.  Memory: one pass holds MC_ROWS_PER_PASS replicated
    inputs plus the model's activations for them — 8192 rows of 28 x 28 float32 are 26 MB, but of 3 x 224 x 224
    3.9 GB before any activation; for large inputs pass a smaller `batch_size`, or a `sample_size` that keeps
    batch_size x sample_size small (a batch is never split, so batch_size rows is the floor).  The passes draw
    from torch's RNG seeded with `seed` inside `torch.random.fork_rng` (forking only the host's and the model
    device's state), so results repeat and the caller's RNG state is untouched.

    sampler: None reads the B200TIP_MC environment variable, default "torch" (the MC-dropout passes above).
    "head" samples only the model's head from its first top-level dropout child on (`mc_head_layers`; ValueError
    for a model it cannot sample, before any work): the point pass captures the head's input (2-D float32 [N, D]),
    and `tip_mc_head` draws the masks and runs the dense layers for all `sample_size` samples of MC_ROWS_PER_PASS
    rows per launch, fed to the same vote kernels.  Its masks are this library's counter-based draws keyed by
    (seed, layer, row, sample, unit), not torch's, and dropouts nested in the trunk (the IMDB transformer block's)
    are not sampled, as in uncertainty-wizard; times["VR"] = [0, head-kernel time, vote time, 0]."""
    return _pred_and_uncertainty(model, x, batch_size, sample_size, [seed], sampler, stacked=False)[0]


def get_pred_and_uncertainty_stack(stack, x, batch_size: int = 32, sample_size: int = DROPOUT_SAMPLE_SIZE,
                                   seeds: Optional[Sequence[int]] = None, sampler: Optional[str] = None
                                   ) -> List[Tuple[np.ndarray, Dict[str, np.ndarray], Dict[str, List[float]]]]:
    """`get_pred_and_uncertainty` for the M models of a `StackedSequential` (`case_studies.stacked.stack`) on the
    same inputs x: one (pred, uncertainties, times) triple per model, in stack order, each in the form
    `get_pred_and_uncertainty` returns.

    The point pass is one stacked forward per batch of `batch_size` inputs (the batch repeated for every model in the
    stack's input layout), and max softmax, PCS, softmax entropy and DeepGini each run once over the [M * N, C]
    probabilities.  seeds: M ints, None = M zeros (each model's `seed` of `get_pred_and_uncertainty`).

    sampler as in `get_pred_and_uncertainty`.  "head": the point pass captures the head's input [M, B, D] from the
    stack (`mc_head_layers_stack`) and `tip_mc_head_stack` samples every model's head, model m's masks keyed by
    seeds[m] exactly as `tip_mc_head` keys a single model's, in launches of MC_ROWS_PER_PASS model-rows; the votes
    go to one `Votes` over the M * N rows.  "torch": the stack's own dropout modules in training mode, on batches
    replicated up to MC_ROWS_PER_PASS model-rows per pass, drawing from torch's RNG seeded once with seeds[0]: every
    model gets its own masks (dropout acts element-wise on the stacked tensor, as in `fit_stack`), which are not the
    masks `get_pred_and_uncertainty` would draw for that model alone.

    times: each phase is timed once for the whole stack and split evenly, so times[name] = [0, prediction time / M,
    quantifier time / M, 0] (for "VR": sampling and vote time / M).  Every module's mode is restored afterwards.
    ValueError, before any work, for a module that is not a StackedSequential, a seed count other than M, an
    unknown sampler, a head the head sampler cannot sample, or an empty x."""
    from ..case_studies.stacked import StackedSequential

    if not isinstance(stack, StackedSequential):
        raise ValueError(f"get_pred_and_uncertainty_stack takes a StackedSequential, got {type(stack).__name__}")
    n_models = len(stack.sources)
    seeds = [0] * n_models if seeds is None else [int(s) for s in seeds]
    if len(seeds) != n_models:
        raise ValueError(f"{len(seeds)} seeds for a stack of {n_models} models")
    return _pred_and_uncertainty(stack, x, batch_size, sample_size, seeds, sampler, stacked=True)


def _pred_and_uncertainty(model, x, batch_size: int, sample_size: int, seeds: List[int], sampler: Optional[str],
                          stacked: bool) -> List[Tuple[np.ndarray, Dict[str, np.ndarray], Dict[str, List[float]]]]:
    """What `get_pred_and_uncertainty` and `get_pred_and_uncertainty_stack` compute, for M = len(seeds) models in the
    [M, N, C] layout: the M models of a StackedSequential when `stacked`, else one model (M = 1) whose outputs gain a
    leading axis.  Returns one (pred, uncertainties, times) triple per model, each phase's time split evenly over
    the M models."""
    import torch
    from torch.nn.modules.dropout import _DropoutNd

    from . import quantifiers as Q
    from .deepgini import DeepGini
    from .timer import Timer
    from .. import engine as E

    sampler = sampler if sampler is not None else os.environ.get("B200TIP_MC", "torch")
    if sampler not in MC_SAMPLERS:
        raise ValueError(f"sampler must be one of {MC_SAMPLERS}, got {sampler!r}")
    head_at, head = (mc_head_layers_stack if stacked else mc_head_layers)(model) if sampler == "head" else (-1, [])
    score_dev = E.require_cuda()
    dev = next(iter(model.parameters()), torch.empty(0)).device
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if x.shape[0] == 0:
        raise ValueError("x holds no inputs")
    x = x.to(dev)
    n, n_models = x.shape[0], len(seeds)

    def forward(xb):
        """every model's output on the batch xb, [M, b, C]"""
        if stacked:
            return model(model.stack_inputs([xb] * n_models)).detach()
        return model(xb).detach()[None]

    def point_pass():
        with torch.no_grad():
            outs = [forward(x[start:start + batch_size]) for start in range(0, n, batch_size)]
        return torch.cat(outs, dim=1) if len(outs) != 1 else outs[0]

    modes = [(m, m.training) for m in model.modules()]
    uncertainties: List[Dict[str, np.ndarray]] = [{} for _ in range(n_models)]
    times: List[Dict[str, List[float]]] = [{} for _ in range(n_models)]
    trunk: List[torch.Tensor] = []
    hook = (list(model.children())[head_at].register_forward_pre_hook(lambda _m, inp: trunk.append(inp[0].detach()))
            if head else None)
    try:
        model.eval()
        pred_timer = Timer()
        try:
            probs = _synced(point_pass, pred_timer, score_dev, dev)
        finally:
            if hook is not None:
                hook.remove()
        if probs.dim() != 3 or probs.shape[:2] != (n_models, n):
            raise ValueError(f"the model returned {tuple(probs.shape)}, expected [{n_models}, {n}, classes]")
        c = probs.shape[2]
        flat = probs.reshape(n_models * n, c)
        pred = None
        for q in (Q.MaxSoftmax, Q.PredictionConfidenceScore, Q.SoftmaxEntropy, DeepGini):
            timer = Timer()
            q_pred, values = _synced(lambda: q.calculate(flat), timer, score_dev, dev)
            if pred is None:
                pred = q_pred.reshape(n_models, n)
            name = q.aliases()[0].replace("custom::", "")
            values = q.cast_conf_or_unc(False, values).reshape(n_models, n)
            for m in range(n_models):
                uncertainties[m][name] = values[m]
                times[m][name] = [0, pred_timer.get() / n_models, timer.get() / n_models, 0]

        dropouts = [m for m in model.modules() if isinstance(m, _DropoutNd)]
        if head or dropouts:
            votes = Q.Votes(n_models * n, c, score_dev)
            sampling_timer, vote_timer = Timer(), Timer()

            def vote(out, samples, start, rows):
                # out [M, rows, samples, C] (or its [M, rows * samples, C] view); model m's rows are votes rows m * n + i
                for m in range(n_models):
                    votes.add(out[m], samples, sample_stride=c, row_stride=samples * c, row0=m * n + start, rows=rows)

            if head:
                h = E.to_device(head_input(trunk, n, n_models) if stacked else head_input(trunk, n)[None], score_dev)
                layers = _head_tensors(head, score_dev)
                rows_per_pass = max(1, MC_ROWS_PER_PASS // n_models)
                for start in range(0, n if sample_size >= 1 else 0, rows_per_pass):
                    b = min(rows_per_pass, n - start)

                    def sample():
                        if stacked:
                            return E.mc_head_stack(h[:, start:start + b], layers, seeds, sample_size, row0=start)
                        return E.mc_head(h[0, start:start + b], layers, seeds[0], sample_size, row0=start)[None]
                    out = _synced(sample, sampling_timer, score_dev, dev)
                    if out.shape[3] != c:
                        raise ValueError(f"the head gives {out.shape[3]} classes, the model's output {c}")
                    _synced(lambda: vote(out, sample_size, start, b), vote_timer, score_dev, dev)
            else:
                for m in dropouts:
                    m.train()
                with torch.random.fork_rng(devices=[dev] if dev.type == "cuda" else []), torch.no_grad():
                    torch.default_generator.manual_seed(seeds[0])
                    if dev.type == "cuda":
                        with torch.cuda.device(dev):
                            torch.cuda.manual_seed(seeds[0])
                    for start in range(0, n, batch_size):
                        xb = x[start:start + batch_size]
                        b = xb.shape[0]
                        done = 0
                        while done < sample_size:
                            r = min(sample_size - done, max(1, MC_ROWS_PER_PASS // (b * n_models)))
                            # row i * r + j of a model's pass is replica j of input i: [b, r, C] once viewed
                            xr = xb.unsqueeze(1).expand(b, r, *xb.shape[1:]).reshape(b * r, *xb.shape[1:])
                            out = _synced(lambda: forward(xr), sampling_timer, score_dev, dev)
                            if tuple(out.shape) != (n_models, b * r, c):
                                raise ValueError(f"an MC-dropout pass returned {tuple(out.shape)}, expected "
                                                 f"{(n_models, b * r, c)}")
                            o = out if out.dtype in (torch.float32, torch.float64) else out.to(torch.float32)
                            _synced(lambda: vote(E.to_device(o, score_dev), r, start, b), vote_timer, score_dev, dev)
                            done += r
            _, vr = _synced(lambda: votes.finish(sample_size), vote_timer, score_dev, dev)
            vr = vr.reshape(n_models, n)
            for m in range(n_models):
                uncertainties[m]["VR"] = vr[m]
                times[m]["VR"] = [0, sampling_timer.get() / n_models, vote_timer.get() / n_models, 0]
    finally:
        for m, training in modes:
            m.training = training
    return [(pred[m], uncertainties[m], times[m]) for m in range(n_models)]


def _badge_dir(root: str, case_study: str, model_id: int, dataset: str) -> str:
    return os.path.join(root, "activations", case_study, f"model_{model_id}", dataset)


def persist_badge(root: str, case_study: str, model_id: int, dataset: str, badge_id: int, activations: Sequence,
                  labels) -> None:
    """One badge in the reference's layout (activation_persistor.py:13-35; `root` is "/assets" there)."""
    path = _badge_dir(root, case_study, model_id, dataset)
    for layer_i, layer_at in enumerate(activations):
        folder = os.path.join(path, f"layer_{layer_i}")
        os.makedirs(folder, exist_ok=True)
        np.save(os.path.join(folder, f"badge_{badge_id}.npy"), _to_numpy(layer_at))
    folder = os.path.join(path, "labels")
    os.makedirs(folder, exist_ok=True)
    np.save(os.path.join(folder, f"badge_{badge_id}.npy"), _to_numpy(labels))


def persist_badges(root: str, case_study: str, model_id: int, dataset: str, transparent_model: TransparentModel, x, y,
                   badge_size: int = BADGE_SIZE) -> int:
    """Walks (x, y) in badges and persists every layer's activations; returns the number of badges
    (activation_persistor.py:52-72)."""
    n_badges = 0
    for badge_id, start in enumerate(range(0, x.shape[0], badge_size)):
        acts = transparent_model.get_activations(x[start:start + badge_size])
        persist_badge(root, case_study, model_id, dataset, badge_id, acts, y[start:start + badge_size])
        n_badges += 1
    return n_badges


def load_badges(root: str, case_study: str, model_id: int, dataset: str, layers: Optional[Sequence[int]] = None
                ) -> Tuple[List[np.ndarray], np.ndarray]:
    """Reads a persisted dataset back: (one [N, ...] array per layer, labels [N]), badges in order."""
    path = _badge_dir(root, case_study, model_id, dataset)
    if layers is None:
        layers = sorted(int(f.split("_")[1]) for f in os.listdir(path) if f.startswith("layer_"))
    label_dir = os.path.join(path, "labels")
    badge_ids = sorted(int(f[len("badge_"):-len(".npy")]) for f in os.listdir(label_dir) if f.endswith(".npy"))
    labels = np.concatenate([np.load(os.path.join(label_dir, f"badge_{b}.npy")) for b in badge_ids])
    acts = [np.concatenate([np.load(os.path.join(path, f"layer_{layer}", f"badge_{b}.npy")) for b in badge_ids])
            for layer in layers]
    return acts, labels


def _to_numpy(a) -> np.ndarray:
    if isinstance(a, np.ndarray):
        return a
    try:
        import torch

        if isinstance(a, torch.Tensor):
            return a.detach().cpu().numpy()
    except ImportError:      # pragma: no cover
        pass
    return np.asarray(a)
