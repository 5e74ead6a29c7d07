"""M networks of one architecture as one module, so that they take their training steps together.

`stack(models)` builds, from M `KerasSequential` networks of one architecture, a `StackedSequential` whose layers
compute all M models at once: each Conv2D becomes one grouped convolution (groups = M) on an NHWC tensor of M * C
channels, each Dense one batched GEMM with kernel [M, in, out], the embedding one lookup into an [M * V, E] table,
the attention's projections batched GEMMs and its attention one SDPA call over M * B sequences.  Every stacked
parameter is the M models' parameters of the same name stacked on a new leading axis, so `unstack()` writes model
m's parameters back as `p[m]`, bit for bit.

Layouts: a stack whose first layer is a Conv2D or MaxPooling2D takes its input channel-interleaved, [B, H, W, M * C]
with channel m * C + c = model m's channel c (`tip_stack_gather`'s interleaved layout), and keeps that layout up to
its Flatten; every other stack takes its input model-major, [M, B, ...].  `model_major(child, y)` turns any child's
output back into [M, B, ...], so callers that read hooked layers never re-derive these layouts.  `logits(x)` returns
[M, B, classes], contiguous, the input of `tip_softmax_xent_seg`.  Dropout acts element-wise on the stacked tensor, so each model
draws its own mask.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F

from ..core.training import keras_initialize
from .base import (Conv2D, Dense, Flatten, GlobalAveragePooling1D, InputLayer, KerasSequential, MaxPooling2D,
                   MultiHeadAttention, TokenAndPositionEmbedding, TransformerBlock)


def _param(src: torch.nn.Module, name: str, models: int) -> torch.nn.Parameter:
    """A placeholder of the stacked shape of `src`'s parameter `name`; `stack` fills it."""
    p = getattr(src, name)
    return torch.nn.Parameter(torch.empty((models, *p.shape), dtype=p.dtype, device=p.device))


def _activate(y, activation):
    if activation == "relu":
        return F.relu(y)
    if activation == "softmax":
        return F.softmax(y, dim=-1)
    return y


class StackedConv2D(torch.nn.Module):
    """M Conv2D layers as one `F.conv2d(groups=M)` on [B, H, W, M * Ci] tensors: weight [M, Co, Ci, kh, kw]."""

    def __init__(self, src: Conv2D, models: int):
        super().__init__()
        self.activation = src.activation
        self.weight, self.bias = _param(src, "weight", models), _param(src, "bias", models)

    def forward(self, x):
        x = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)     # a view of NHWC input
        m, co = self.weight.shape[:2]
        y = F.conv2d(x, self.weight.reshape(m * co, *self.weight.shape[2:]), self.bias.reshape(m * co), groups=m)
        return _activate(y, self.activation).permute(0, 2, 3, 1)


class StackedFlatten(torch.nn.Module):
    """Flatten per model: [B, H, W, M * C] (interleaved) or [M, B, ...] (model-major) to [M, B, features], each model
    in Keras' row-major (H, W, C) order."""

    def __init__(self, models: int, interleaved: bool):
        super().__init__()
        self.models, self.interleaved = models, interleaved

    def forward(self, x):
        if not self.interleaved:
            return x.reshape(x.shape[0], x.shape[1], -1)
        b, h, w, mc = x.shape
        return x.reshape(b, h, w, self.models, mc // self.models).permute(3, 0, 1, 2, 4).reshape(self.models, b, -1)


class StackedDense(torch.nn.Module):
    """M Dense layers as one `baddbmm` over [M, rows, in]: kernel [M, in, out], bias [M, out]; inputs [M, ..., in]."""

    def __init__(self, src: Dense, models: int):
        super().__init__()
        self.activation = src.activation
        self.kernel, self.bias = _param(src, "kernel", models), _param(src, "bias", models)

    def logits(self, x):
        m, i, o = self.kernel.shape
        y = torch.baddbmm(self.bias.unsqueeze(1), x.reshape(m, -1, i), self.kernel)
        return y.reshape(*x.shape[:-1], o)

    def forward(self, x):
        return _activate(self.logits(x), self.activation)


class StackedTokenAndPositionEmbedding(torch.nn.Module):
    """M embeddings as one lookup: ids [M, B, L] + m * V into the [M * V, E] view of token_emb [M, V, E]."""

    def __init__(self, src: TokenAndPositionEmbedding, models: int):
        super().__init__()
        self.token_emb, self.pos_emb = _param(src, "token_emb", models), _param(src, "pos_emb", models)

    def forward(self, x):
        m, v, e = self.token_emb.shape
        offset = torch.arange(m, dtype=torch.int64, device=x.device).mul_(v).view(m, *([1] * (x.dim() - 1)))
        ids = x.to(torch.int64) + offset
        return F.embedding(ids, self.token_emb.reshape(m * v, e)) + self.pos_emb[:, None, :ids.shape[-1]]


class StackedMultiHeadAttention(torch.nn.Module):
    """M self-attention layers: the projections as bmm over [M, B * L, E], the attention one SDPA over
    [M * B, heads, L, key_dim]."""

    NAMES = ("query", "key", "value", "output")

    def __init__(self, src: MultiHeadAttention, models: int):
        super().__init__()
        for name in self.NAMES:
            for part in ("kernel", "bias"):
                self.register_parameter(f"{name}_{part}", _param(src, f"{name}_{part}", models))

    def _project(self, x, name):
        # [M, B, L, E] x [M, E, H, D] -> [M * B, H, L, D]
        k, b = getattr(self, f"{name}_kernel"), getattr(self, f"{name}_bias")
        m, e, h, d = k.shape
        y = torch.baddbmm(b.reshape(m, 1, h * d), x.reshape(m, -1, e), k.reshape(m, e, h * d))
        return y.view(m * x.shape[1], x.shape[2], h, d).transpose(1, 2)

    def forward(self, x):
        q, k, v = (self._project(x, n) for n in ("query", "key", "value"))
        o = F.scaled_dot_product_attention(q, k, v)
        m, h, d, e = self.output_kernel.shape
        o = o.transpose(1, 2).reshape(m, -1, h * d)
        y = torch.baddbmm(self.output_bias.unsqueeze(1), o, self.output_kernel.reshape(m, h * d, e))
        return y.view(x.shape)


class StackedLayerNorm(torch.nn.Module):
    """M LayerNorms over the last axis: the normalisation without affine, then each model's weight and bias."""

    def __init__(self, src: torch.nn.LayerNorm, models: int):
        super().__init__()
        self.normalized_shape, self.eps = tuple(src.normalized_shape), src.eps
        self.weight, self.bias = _param(src, "weight", models), _param(src, "bias", models)

    def forward(self, x):
        shape = (self.weight.shape[0],) + (1,) * (x.dim() - 1 - len(self.normalized_shape)) + self.normalized_shape
        y = F.layer_norm(x, self.normalized_shape, eps=self.eps)
        return torch.addcmul(self.bias.view(shape), y, self.weight.view(shape))


class StackedTransformerBlock(torch.nn.Module):
    """TransformerBlock on [M, B, L, E], with the block's submodule names (so its parameters keep theirs)."""

    def __init__(self, src: TransformerBlock, models: int):
        super().__init__()
        self.att = StackedMultiHeadAttention(src.att, models)
        self.ffn = torch.nn.Sequential(*(StackedDense(d, models) for d in src.ffn))
        self.layernorm1 = StackedLayerNorm(src.layernorm1, models)
        self.layernorm2 = StackedLayerNorm(src.layernorm2, models)
        self.dropout1 = torch.nn.Dropout(src.dropout1.p)
        self.dropout2 = torch.nn.Dropout(src.dropout2.p)

    forward = TransformerBlock.forward


class StackedGlobalAveragePooling1D(torch.nn.Module):
    def forward(self, x):                   # [M, B, L, E] -> [M, B, E]
        return x.mean(dim=2)


def _stacked_layer(layer: torch.nn.Module, models: int, interleaved: bool) -> torch.nn.Module:
    if isinstance(layer, Conv2D):
        return StackedConv2D(layer, models)
    if isinstance(layer, Dense):
        return StackedDense(layer, models)
    if isinstance(layer, MaxPooling2D):
        return MaxPooling2D(layer.pool_size)
    if isinstance(layer, Flatten):
        return StackedFlatten(models, interleaved)
    if isinstance(layer, torch.nn.Dropout):
        return torch.nn.Dropout(layer.p)
    if isinstance(layer, InputLayer):
        return InputLayer()
    if isinstance(layer, TokenAndPositionEmbedding):
        return StackedTokenAndPositionEmbedding(layer, models)
    if isinstance(layer, TransformerBlock):
        return StackedTransformerBlock(layer, models)
    if isinstance(layer, GlobalAveragePooling1D):
        return StackedGlobalAveragePooling1D()
    raise TypeError(f"stack cannot stack a {type(layer).__module__}.{type(layer).__qualname__} layer")


class StackedSequential(torch.nn.Sequential):
    """M `KerasSequential` networks as one (see the module docstring); built by `stack`."""

    def __init__(self, models: Sequence[KerasSequential]):
        first = list(models[0].children())
        interleaved = bool(first) and isinstance(first[0], (Conv2D, MaxPooling2D))
        super().__init__(*(_stacked_layer(layer, len(models), interleaved) for layer in first))
        self.channels_interleaved, self.cast_input = interleaved, models[0].cast_input
        self.__dict__["sources"] = list(models)       # not submodules: their parameters are not the stack's

    def stack_inputs(self, xs: Sequence[torch.Tensor]) -> torch.Tensor:
        """The stacked input of per-model inputs xs[m] (each [B, ...]) in this stack's layout."""
        if self.channels_interleaved:
            x = torch.stack(list(xs), dim=3)                     # [B, H, W, M, C]
            return x.reshape(*x.shape[:3], -1)
        return torch.stack(list(xs))

    def model_major(self, child: int, y: torch.Tensor) -> torch.Tensor:
        """The output y of child `child` as [M, B, *model m's layer shape], slice m being what model m's own layer
        gives: the inverse of `stack_inputs` for that child's layout.  Children before the Flatten of an
        interleaved stack give [B, H, W, M * C] (returned as a strided view); every other child gives [M, B, ...]
        (returned as is).  IndexError for a child index out of range."""
        children = list(self.children())
        if not 0 <= child < len(children):
            raise IndexError(f"child index {child} out of range (the stack has {len(children)} children)")
        flatten_at = next((i for i, c in enumerate(children) if isinstance(c, StackedFlatten)), len(children))
        if self.channels_interleaved and child < flatten_at:
            m = len(self.sources)
            b, h, w, mc = y.shape
            return y.reshape(b, h, w, m, mc // m).permute(3, 0, 1, 2, 4)
        return y

    def logits(self, x):
        x = x.to(torch.float32) if self.cast_input else x
        layers = list(self.children())
        for layer in layers[:-1]:
            x = layer(x)
        return layers[-1].logits(x).contiguous()

    def forward(self, x):
        return super().forward(x.to(torch.float32) if self.cast_input else x)

    def unstack(self) -> List[KerasSequential]:
        """Copies every stacked parameter's slice m into model m's parameter of the same name; returns the models."""
        with torch.no_grad():
            for name, p in self.named_parameters():
                for m, model in enumerate(self.sources):
                    model.get_parameter(name).copy_(p[m])
        return self.sources


def stack(models: Sequence[KerasSequential], seeds: Optional[Sequence[int]] = None) -> StackedSequential:
    """One `StackedSequential` of M >= 1 networks of one architecture, its parameters copied from theirs.

    seeds: None keeps the models' weights; M ints first re-initialise model k with Keras' initialisers from a host
    generator seeded with seeds[k] (what `fit(seed=seeds[k])` does).  ValueError when the models differ in a layer's
    class or a parameter's shape, TypeError (naming it) for a layer type that has no stacked form."""
    models = list(models)
    if not models:
        raise ValueError("stack takes at least one model")
    if not all(isinstance(m, KerasSequential) for m in models):
        bad = next(m for m in models if not isinstance(m, KerasSequential))
        raise TypeError(f"stack takes KerasSequential networks, not {type(bad).__qualname__}")
    if seeds is not None and len(seeds) != len(models):
        raise ValueError(f"{len(seeds)} seeds for {len(models)} models")
    ref = models[0]
    ref_layers = [type(c) for c in ref.modules()]
    ref_params = [(n, p.shape) for n, p in ref.named_parameters()]
    for k, m in enumerate(models[1:], start=1):
        if [type(c) for c in m.modules()] != ref_layers or m.cast_input != ref.cast_input:
            raise ValueError(f"model {k}'s layers differ from model 0's")
        if [(n, p.shape) for n, p in m.named_parameters()] != ref_params:
            raise ValueError(f"model {k}'s parameters differ in name or shape from model 0's")
        if any(a.training != b.training or getattr(a, "p", None) != getattr(b, "p", None)
               for a, b in zip(ref.modules(), m.modules())):
            raise ValueError(f"model {k}'s modes or dropout rates differ from model 0's")
    if seeds is not None:
        for m, seed in zip(models, seeds):
            keras_initialize(m, torch.Generator().manual_seed(int(seed)))
    net = StackedSequential(models)
    with torch.no_grad():
        for name, p in net.named_parameters():
            p.copy_(torch.stack([m.get_parameter(name).detach() for m in models]))
    return net.train(ref.training)
