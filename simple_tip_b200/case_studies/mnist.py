"""The MNIST case study (case_study_mnist.py): the Keras example's CNN, 15 epochs of batch 128, MNIST-C as the
corrupted set."""
from __future__ import annotations

import os

import numpy as np
import torch

from .base import CaseStudy, Conv2D, Dense, Flatten, KerasSequential, MaxPooling2D

NAME = "mnist"
SA_ACTIVATION_LAYERS = [3]
NC_ACTIVATION_LAYERS = [0, 1, 2, 3]
PREDICTION_BADGE_SIZE = 128
OOD_FILES = ("mnist_c_images.npy", "mnist_c_labels.npy")


def network() -> KerasSequential:
    """case_study_mnist.py:51-62; children = Keras' model.layers (the Input is not a layer of a Sequential)."""
    return KerasSequential(
        Conv2D(1, 32, 3, "relu"), MaxPooling2D(2), Conv2D(32, 64, 3, "relu"), MaxPooling2D(2), Flatten(),
        torch.nn.Dropout(0.5), Dense(5 * 5 * 64, 10, "softmax"))


def load_datasets(nominal, datasets_folder: str):
    """`_load_datasets` (case_study_mnist.py:153-166).  nominal = ((x_train, y_train), (x_test, y_test)) as
    `tf.keras.datasets.mnist.load_data()` returns them (uint8 images [N, 28, 28]); MNIST-C from `datasets_folder`."""
    (x_train, y_train), (x_test, y_test) = nominal
    x_test = np.expand_dims(x_test, -1).astype("float32") / 255.0
    x_train = np.expand_dims(x_train, -1).astype("float32") / 255.0
    ood_x_test = np.load(os.path.join(datasets_folder, OOD_FILES[0])).astype("float32") / 255.0
    ood_y_test = np.load(os.path.join(datasets_folder, OOD_FILES[1]))

    ood_x_test = np.concatenate((x_test, ood_x_test), axis=0)
    ood_y_test = np.concatenate((y_test, ood_y_test), axis=0)
    shuffle_args = np.random.default_rng(0).permutation(len(ood_y_test))
    return (x_train, y_train), (x_test, y_test), (ood_x_test[shuffle_args], ood_y_test[shuffle_args])


class MnistCaseStudy(CaseStudy):
    name = NAME
    num_classes = 10
    batch_size = 128
    epochs = 15
    sa_layers = SA_ACTIVATION_LAYERS
    nc_layers = NC_ACTIVATION_LAYERS
    num_selected = 1000
    prediction_badge_size = PREDICTION_BADGE_SIZE
    network = staticmethod(network)
