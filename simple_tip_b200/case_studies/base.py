"""What the four case studies share (case_study.py:13-144): Keras' layers as torch modules, and the runner.

The networks are `KerasSequential` modules whose `children()` are, index for index, Keras' `model.layers`, so the
integer layer ids of `TransparentModel` (and with it of both experiments' arms) mean what the reference's
`SA_ACTIVATION_LAYERS` / `NC_ACTIVATION_LAYERS` mean.  Conv2D and Dense carry their activation, as in Keras; image
layers take and return NHWC tensors (Keras' `channels_last`), so traces and persisted badges have Keras' shapes: the
convolutions run on the NHWC tensor viewed as NCHW, which torch executes in its channels_last memory format, and
the view back is free.  Kernels are stored in Keras' layouts where torch does not prescribe one (Dense [in, out],
the attention projections [embed, heads, key_dim] / [heads, key_dim, embed]), Conv2D in torch's [out, in, kh, kw].

`CaseStudy` runs the reference's four phases for a torch model — `train`, `run_prio_eval`,
`run_active_learning_eval`, `collect_activations` — over an output folder, one model after the other (uwiz's
process pool and its `context` are not part of it).  `train` and `run_active_learning_eval` can instead train their
models together in one stack (`stacked=True`, `core.training.fit_stack`), in one process on one GPU, and
`run_prio_eval(stacked=True)` scores the fault predictors of a stack of models in one pass.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from ..core import active_learning, activations, prioritization
from ..core.training import fit, fit_stack, glorot_limit, uniform_

MODELS_FOLDER = "models"


def model_path(output_folder: str, name: str, model_id: int) -> str:
    """Where `CaseStudy.train` saves a model's state_dict: {output_folder}/models/{name}/model_{id}.pt."""
    return os.path.join(output_folder, MODELS_FOLDER, name, f"model_{model_id}.pt")


def load_state(model: torch.nn.Module, path: str, device) -> torch.nn.Module:
    model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))
    return model.to(device).eval()


def _zeros_(t):
    with torch.no_grad():
        t.zero_()


def _glorot_(t, keras_shape, generator):
    uniform_(t, glorot_limit(keras_shape), generator)


class Conv2D(torch.nn.Module):
    """tf.keras.layers.Conv2D(filters, kernel_size, activation) with 'valid' padding, stride 1, on NHWC tensors."""

    def __init__(self, in_channels: int, filters: int, kernel_size: int, activation: Optional[str] = None):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(filters, in_channels, kernel_size, kernel_size))
        self.bias = torch.nn.Parameter(torch.empty(filters))
        self.activation = activation
        self.keras_init(None)

    def keras_init(self, generator):
        co, ci, kh, kw = self.weight.shape
        _glorot_(self.weight, (kh, kw, ci, co), generator)
        _zeros_(self.bias)

    def forward(self, x):
        x = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)     # a view of NHWC input
        y = F.conv2d(x, self.weight, self.bias)
        if self.activation == "relu":
            y = F.relu(y)
        return y.permute(0, 2, 3, 1)


class MaxPooling2D(torch.nn.Module):
    """tf.keras.layers.MaxPooling2D(pool_size) ('valid', strides = pool_size) on NHWC tensors."""

    def __init__(self, pool_size: int):
        super().__init__()
        self.pool_size = pool_size

    def forward(self, x):
        x = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        return F.max_pool2d(x, self.pool_size).permute(0, 2, 3, 1)


class Flatten(torch.nn.Module):
    """tf.keras.layers.Flatten: row-major over Keras' (H, W, C)."""

    def forward(self, x):
        return x.reshape(x.shape[0], -1)


class Dense(torch.nn.Module):
    """tf.keras.layers.Dense(units, activation) on the last axis; kernel [in, units] as Keras stores it.
    `logits(x)` is the layer before its activation."""

    def __init__(self, in_features: int, units: int, activation: Optional[str] = None):
        super().__init__()
        self.kernel = torch.nn.Parameter(torch.empty(in_features, units))
        self.bias = torch.nn.Parameter(torch.empty(units))
        self.activation = activation
        self.keras_init(None)

    def keras_init(self, generator):
        _glorot_(self.kernel, self.kernel.shape, generator)
        _zeros_(self.bias)

    def logits(self, x):
        if x.dim() == 2:
            return torch.addmm(self.bias, x, self.kernel)
        return torch.matmul(x, self.kernel) + self.bias

    def forward(self, x):
        y = self.logits(x)
        if self.activation == "relu":
            return F.relu(y)
        if self.activation == "softmax":
            return F.softmax(y, dim=-1)
        return y


class InputLayer(torch.nn.Module):
    """The functional model's tf.keras.layers.Input(shape) layer: its float32 input, as Keras casts it."""

    def forward(self, x):
        return x.to(torch.float32)


class TokenAndPositionEmbedding(torch.nn.Module):
    """case_study_imdb.py:118-149: token embedding + position embedding (tf.keras.layers.Embedding, initialised
    U(-0.05, 0.05)); ids arrive as floats, as Keras' Input hands them over, and are cast to integers."""

    def __init__(self, maxlen: int, vocab_size: int, embed_dim: int):
        super().__init__()
        self.token_emb = torch.nn.Parameter(torch.empty(vocab_size, embed_dim))
        self.pos_emb = torch.nn.Parameter(torch.empty(maxlen, embed_dim))
        self.keras_init(None)

    def keras_init(self, generator):
        uniform_(self.token_emb, 0.05, generator)
        uniform_(self.pos_emb, 0.05, generator)

    def forward(self, x):
        ids = x.to(torch.int64)
        return F.embedding(ids, self.token_emb) + self.pos_emb[:ids.shape[-1]]


class MultiHeadAttention(torch.nn.Module):
    """tf.keras.layers.MultiHeadAttention(num_heads, key_dim) self-attention (no mask, attention dropout 0): the
    query / key / value EinsumDense kernels [embed, heads, key_dim] with biases [heads, key_dim], the output kernel
    [heads, key_dim, embed] with bias [embed], all glorot_uniform with Keras' fans (fan_in = heads * embed,
    fan_out = key_dim * embed for the projections); scaled dot-product attention by torch."""

    def __init__(self, embed_dim: int, num_heads: int, key_dim: int):
        super().__init__()
        for name in ("query", "key", "value"):
            self.register_parameter(f"{name}_kernel", torch.nn.Parameter(torch.empty(embed_dim, num_heads, key_dim)))
            self.register_parameter(f"{name}_bias", torch.nn.Parameter(torch.empty(num_heads, key_dim)))
        self.output_kernel = torch.nn.Parameter(torch.empty(num_heads, key_dim, embed_dim))
        self.output_bias = torch.nn.Parameter(torch.empty(embed_dim))
        self.keras_init(None)

    def keras_init(self, generator):
        for name in ("query", "key", "value", "output"):
            k = getattr(self, f"{name}_kernel")
            _glorot_(k, k.shape, generator)
            _zeros_(getattr(self, f"{name}_bias"))

    def _project(self, x, name):
        # [B, T, E] x [E, H, D] -> [B, H, T, D]
        k, b = getattr(self, f"{name}_kernel"), getattr(self, f"{name}_bias")
        e, h, d = k.shape
        return (torch.matmul(x, k.reshape(e, h * d)) + b.reshape(h * d)).view(*x.shape[:2], h, d).transpose(1, 2)

    def forward(self, x):
        q, k, v = (self._project(x, n) for n in ("query", "key", "value"))
        o = F.scaled_dot_product_attention(q, k, v)                      # softmax(q k^T / sqrt(key_dim)) v
        h, d, e = self.output_kernel.shape
        o = o.transpose(1, 2).reshape(*x.shape[:2], h * d)
        return torch.matmul(o, self.output_kernel.reshape(h * d, e)) + self.output_bias


class TransformerBlock(torch.nn.Module):
    """case_study_imdb.py:48-80: attention, dropout, residual + LayerNorm, feed-forward (Dense relu, Dense),
    dropout, residual + LayerNorm (epsilon 1e-6)."""

    def __init__(self, embed_dim: int, num_heads: int, ff_dim: int, rate: float = 0.1):
        super().__init__()
        self.att = MultiHeadAttention(embed_dim, num_heads, embed_dim)
        self.ffn = torch.nn.Sequential(Dense(embed_dim, ff_dim, "relu"), Dense(ff_dim, embed_dim))
        self.layernorm1 = torch.nn.LayerNorm(embed_dim, eps=1e-6)
        self.layernorm2 = torch.nn.LayerNorm(embed_dim, eps=1e-6)
        self.dropout1 = torch.nn.Dropout(rate)
        self.dropout2 = torch.nn.Dropout(rate)

    def keras_init(self, generator):
        for ln in (self.layernorm1, self.layernorm2):
            with torch.no_grad():
                ln.weight.fill_(1.0)
                ln.bias.zero_()

    def forward(self, x):
        out1 = self.layernorm1(x + self.dropout1(self.att(x)))
        return self.layernorm2(out1 + self.dropout2(self.ffn(out1)))


class GlobalAveragePooling1D(torch.nn.Module):
    def forward(self, x):
        return x.mean(dim=1)


class KerasSequential(torch.nn.Sequential):
    """A Keras model as a chain of children (= `model.layers`).  `forward` casts the input to float32 (as Keras'
    input layer does) and returns the last layer's softmax; `logits` stops before that softmax (training)."""

    def __init__(self, *layers, cast_input: bool = True):
        super().__init__(*layers)
        self.cast_input = cast_input

    def forward(self, x):
        return super().forward(x.to(torch.float32) if self.cast_input else x)

    def logits(self, x):
        x = x.to(torch.float32) if self.cast_input else x
        layers = list(self.children())
        for layer in layers[:-1]:
            x = layer(x)
        return layers[-1].logits(x)


def one_hot(y, num_classes: int, device) -> torch.Tensor:
    """keras.utils.to_categorical(y, num_classes) as a float32 device tensor."""
    y = torch.as_tensor(np.asarray(y).reshape(-1), dtype=torch.int64, device=device)
    return F.one_hot(y, num_classes).to(torch.float32)


Datasets = Tuple[Tuple[np.ndarray, np.ndarray], Tuple[np.ndarray, np.ndarray], Tuple[np.ndarray, np.ndarray]]


class CaseStudy:
    """One case study's runner (case_study.py:77-144) over `output_folder`.

    `datasets` is what the case study's `load_datasets` returns: ((x_train, y_train), (x_test, y_test),
    (ood_x_test, ood_y_test)).  The inputs are moved to the device once; the labels stay host arrays.  `epochs`,
    `num_selected`: None takes the reference's values (tests and quick runs pass smaller ones).  Models are saved as
    `{output_folder}/models/{name}/model_{id}.pt` (the `state_dict`); the experiments' files go where
    `core.prioritization`, `core.active_learning` and `core.activations` put them under the same folder."""

    name: str
    num_classes: int
    batch_size: int                  # model.fit's batch size
    epochs: int                      # model.fit's epochs
    sa_layers: List[int]
    nc_layers: List[int]
    num_selected: int                # active learning
    prediction_badge_size: int       # badges of the arms' forward passes in the prioritization run
    dsa_badge_size: Optional[int] = None

    @staticmethod
    def network() -> KerasSequential:
        raise NotImplementedError

    def __init__(self, output_folder: str, datasets: Datasets, epochs: Optional[int] = None,
                 num_selected: Optional[int] = None, device=None):
        self.output_folder = output_folder
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if epochs is not None:
            self.epochs = epochs
        if num_selected is not None:
            self.num_selected = num_selected
        (x_train, y_train), (x_test, y_test), (ood_x, ood_y) = datasets
        dev = self.device
        self.train_set = (torch.from_numpy(np.ascontiguousarray(x_train)).to(dev), np.asarray(y_train))
        self.nominal_set = (torch.from_numpy(np.ascontiguousarray(x_test)).to(dev), np.asarray(y_test))
        self.ood_set = (torch.from_numpy(np.ascontiguousarray(ood_x)).to(dev), np.asarray(ood_y))

    # ---- the model -------------------------------------------------------------------------------------------
    def new_model(self) -> KerasSequential:
        return self.network().to(self.device)

    def training_process(self, x, y) -> KerasSequential:
        """`_train_new_model(x, y)`: a fresh network fitted with the case study's recipe (also active learning's
        `training_process`)."""
        return fit(self.new_model(), x.to(self.device), y.to(self.device), self.batch_size, self.epochs,
                   validation_split=0.1)

    def stacked_training_process(self, x_pool, y_pool, rows) -> List[KerasSequential]:
        """The recipe for rows.shape[0] fresh networks trained together (`fit_stack`): network k on
        x_pool[rows[k]], y_pool[rows[k]] (active learning's `stacked_training_process`)."""
        dev = self.device
        models = [self.new_model() for _ in range(rows.shape[0])]
        return fit_stack(models, x_pool.to(dev), y_pool.to(dev), rows.to(dev), self.batch_size, self.epochs,
                         validation_split=0.1)

    def model_path(self, model_id: int) -> str:
        return model_path(self.output_folder, self.name, model_id)

    def load_model(self, model_id: int) -> KerasSequential:
        """The network rebuilt from what `train` saved, on the case study's device, in eval mode."""
        return load_state(self.network(), self.model_path(model_id), self.device)

    # ---- the four phases ---------------------------------------------------------------------------------------
    def train(self, model_ids: Sequence[int], stacked: bool = False) -> None:
        """`_model_creator` per id (case_study.py:77-92): the recipe on the training set, saved.  stacked=True trains
        all ids' models together in one stack (`stacked_training_process`) instead of one after the other."""
        x, y = self.train_set
        y = one_hot(y, self.num_classes, self.device)
        if stacked:
            rows = torch.arange(x.shape[0], dtype=torch.int64, device=self.device).expand(len(model_ids), -1)
            models = self.stacked_training_process(x, y, rows.contiguous())
        else:
            models = (self.training_process(x, y) for _ in model_ids)
        for model_id, model in zip(model_ids, models):
            path = self.model_path(model_id)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            torch.save(model.state_dict(), path)

    def run_prio_eval(self, model_ids: Sequence[int], stacked: bool = False, stack_size: Optional[int] = None,
                      stacked_coverage: bool = False) -> Dict[int, dict]:
        """`_prioritization_evaluator` per id: `core.prioritization.evaluate` with the case study's layers and
        badge sizes; returns {model_id: its APFDs}.  stacked=True loads the ids' models and evaluates them in stacks
        of at most `stack_size` (None: all ids in one) with `core.prioritization.evaluate_stack`, which writes the
        same files and scores the fault predictors of a stack in one pass; stacked_coverage=True (only with
        stacked=True, ValueError otherwise) runs each stack's coverage arm together too.  A stacked coverage arm
        holds the stack's test traces, stack_size * N * D * 4 bytes (`StackedCoverageWorker`)."""
        if stacked_coverage and not stacked:
            raise ValueError("stacked_coverage=True needs stacked=True")
        res = {}
        if stacked:
            if stack_size is not None and stack_size < 1:
                raise ValueError(f"stack_size must be >= 1, got {stack_size}")
            ids = list(model_ids)
            size = stack_size or max(len(ids), 1)
            for k in range(0, len(ids), size):
                chunk = ids[k:k + size]
                res.update(prioritization.evaluate_stack(
                    chunk, self.name, [self.load_model(i) for i in chunk], self.train_set[0], self.nominal_set[0],
                    self.nominal_set[1], self.ood_set[0], self.ood_set[1], self.nc_layers, self.sa_layers,
                    dsa_badge_size=self.dsa_badge_size, output_folder=self.output_folder,
                    batch_size=self.prediction_badge_size, stacked_coverage=stacked_coverage))
            return res
        for model_id in model_ids:
            res[model_id] = prioritization.evaluate(
                model_id, self.name, self.load_model(model_id), self.train_set[0], self.nominal_set[0],
                self.nominal_set[1], self.ood_set[0], self.ood_set[1], self.nc_layers, self.sa_layers,
                dsa_badge_size=self.dsa_badge_size, output_folder=self.output_folder,
                batch_size=self.prediction_badge_size)
        return res

    def run_active_learning_eval(self, model_ids: Sequence[int], stacked: bool = False) -> Dict[int, tuple]:
        """`_active_learning_evaluator` per id: `core.active_learning.evaluate` with `training_process` as the
        retraining (stacked=True: a model id's retrainings trained together by `stacked_training_process`); returns
        {model_id: evaluate's result}."""
        res = {}
        for model_id in model_ids:
            res[model_id] = active_learning.evaluate(
                model_id, self.name, self.load_model(model_id), self.train_set[0], self.train_set[1],
                self.nominal_set[0], self.nominal_set[1], self.ood_set[0], self.ood_set[1], self.nc_layers,
                self.sa_layers, self.training_process, observed_share=0.5, num_selected=self.num_selected,
                num_classes=self.num_classes, dsa_badge_size=self.dsa_badge_size, output_folder=self.output_folder,
                stacked_training_process=self.stacked_training_process if stacked else None)
        return res

    def collect_activations(self, model_ids: Sequence[int]) -> None:
        """`_activation_persistor` per id (activation_persistor.persist): every layer's activations, without the
        model output, in badges of 100, for the training, nominal and nominal + corrupted sets."""
        for model_id in model_ids:
            model = self.load_model(model_id)
            layers = list(range(len(list(model.children()))))
            tm = activations.TransparentModel(model, layers, include_last_layer=False)
            for ds, (x, y) in (("train", self.train_set), ("test_nominal", self.nominal_set),
                               ("test_nominal_and_corrupted", self.ood_set)):
                activations.persist_badges(self.output_folder, self.name, model_id, ds, tm, x, y,
                                           activations.BADGE_SIZE)
