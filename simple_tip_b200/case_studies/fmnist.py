"""The Fashion-MNIST case study (case_study_fashion_mnist.py): MNIST's CNN and recipe, FMNIST-C as the corrupted
set."""
from __future__ import annotations

import os

import numpy as np

from . import mnist
from .base import CaseStudy

NAME = "fmnist"
SA_ACTIVATION_LAYERS = [3]
NC_ACTIVATION_LAYERS = [0, 1, 2, 3]
PREDICTION_BADGE_SIZE = 128
OOD_FILES = ("fmnist-c-test.npy", "fmnist-c-test-labels.npy")

network = mnist.network         # case_study_fashion_mnist.py:30-41 is the same network


def load_datasets(nominal, datasets_folder: str):
    """`_load_datasets` (case_study_fashion_mnist.py:134-147).  nominal as `fashion_mnist.load_data()` returns it;
    FMNIST-C ([N, 28, 28] uint8, labels) from `datasets_folder`."""
    (x_train, y_train), (x_test, y_test) = nominal
    x_test = np.expand_dims(x_test, -1).astype("float32") / 255.0
    x_train = np.expand_dims(x_train, -1).astype("float32") / 255.0
    ood_x_test = np.load(os.path.join(datasets_folder, OOD_FILES[0])).astype("float32") / 255.0
    ood_y_test = np.load(os.path.join(datasets_folder, OOD_FILES[1]))

    ood_x_test = np.concatenate((x_test, np.expand_dims(ood_x_test, -1)), axis=0)
    ood_y_test = np.concatenate((y_test, ood_y_test), axis=0)
    shuffle_args = np.random.default_rng(0).permutation(len(ood_y_test))
    return (x_train, y_train), (x_test, y_test), (ood_x_test[shuffle_args], ood_y_test[shuffle_args])


class FashionMnistCaseStudy(CaseStudy):
    name = NAME
    num_classes = 10
    batch_size = 128
    epochs = 15
    sa_layers = SA_ACTIVATION_LAYERS
    nc_layers = NC_ACTIVATION_LAYERS
    num_selected = 1000
    prediction_badge_size = PREDICTION_BADGE_SIZE
    network = staticmethod(network)
