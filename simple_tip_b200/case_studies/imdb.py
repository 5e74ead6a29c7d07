"""The IMDB case study (case_study_imdb.py): the Keras example's one-block transformer classifier, 10 epochs of
batch 32, IMDB-C as the corrupted set; the inputs are `core.imdb`'s five files."""
from __future__ import annotations

import torch

from ..core import imdb as inputs
from .base import (CaseStudy, Dense, GlobalAveragePooling1D, InputLayer, KerasSequential, TokenAndPositionEmbedding,
                   TransformerBlock)

NAME = "imdb"
EMBED_DIM, NUM_HEADS, FF_DIM = 32, 2, 32
SA_ACTIVATION_LAYERS = [5]
# case_study_imdb.py:34-41 as written: sublayer tuples and two layer ids
REFERENCE_NC_ACTIVATION_LAYERS = [
    (1, lambda x: x.token_emb),
    (1, lambda x: x.pos_emb),
    (2, lambda x: x.ffn[0]),
    (2, lambda x: x.ffn[1]),
    3,
    5,
]
BADGE_SIZE = 128


def effective_layers(activation_layers, n_layers: int):
    """The layers the reference's transparent model really hooks (handler_model.py:198-202 keeps `model.layers[i]`
    where `i in activation_layers`): no tuple equals an int, so of the IMDB list only 3 and 5 remain."""
    return [i for i in range(n_layers) if i in activation_layers]


def network() -> KerasSequential:
    """case_study_imdb.py:152-166; children = the functional model's layers, its InputLayer first."""
    return KerasSequential(
        InputLayer(), TokenAndPositionEmbedding(inputs.INPUT_MAXLEN, inputs.VOCAB_SIZE, EMBED_DIM),
        TransformerBlock(EMBED_DIM, NUM_HEADS, FF_DIM), GlobalAveragePooling1D(), torch.nn.Dropout(0.1),
        Dense(EMBED_DIM, 20, "relu"), torch.nn.Dropout(0.1), Dense(20, 2, "softmax"), cast_input=False)


NC_ACTIVATION_LAYERS = effective_layers(REFERENCE_NC_ACTIVATION_LAYERS, 8)

load_datasets = inputs.load_datasets          # case_study_imdb.py:271-285


class ImdbCaseStudy(CaseStudy):
    name = NAME
    num_classes = 2
    batch_size = 32
    epochs = 10
    sa_layers = SA_ACTIVATION_LAYERS
    nc_layers = NC_ACTIVATION_LAYERS
    num_selected = 2500
    prediction_badge_size = BADGE_SIZE
    dsa_badge_size = 500
    network = staticmethod(network)
