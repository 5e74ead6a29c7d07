"""The CIFAR-10 case study (case_study_cifar10.py): the TensorFlow tutorial's CNN with a softmax head, 20 epochs of
batch 32, CIFAR-10-C as the corrupted set."""
from __future__ import annotations

import os

import numpy as np

from .base import CaseStudy, Conv2D, Dense, Flatten, KerasSequential, MaxPooling2D

NAME = "cifar10"
SA_ACTIVATION_LAYERS = [3]
NC_ACTIVATION_LAYERS = [0, 1, 2, 3]
CIFAR_10_BATCH_SIZE = 32
OOD_FILES = ("cifar10_c_images.npy", "cifar10_c_labels.npy")


def network() -> KerasSequential:
    """case_study_cifar10.py:39-49."""
    return KerasSequential(
        Conv2D(3, 32, 3, "relu"), MaxPooling2D(2), Conv2D(32, 64, 3, "relu"), MaxPooling2D(2),
        Conv2D(64, 64, 3, "relu"), Flatten(), Dense(4 * 4 * 64, 64, "relu"), Dense(64, 10, "softmax"))


def prepare_cifar10_c(cifar10_c_folder: str, datasets_folder: str) -> None:
    """`Cifar10CaseStudy._prefetch_datasets` (case_study_cifar10.py:165-208) for an unpacked CIFAR-10-C folder:
    every corruption file concatenated, 10 000 rows chosen by `default_rng(0).permutation`, the labels tiled once
    per file; written to `datasets_folder` unless both files exist.  The files are taken in sorted order (the
    reference takes `os.listdir`'s, which the filesystem decides)."""
    out = [os.path.join(datasets_folder, f) for f in OOD_FILES]
    if all(os.path.exists(p) for p in out):
        return
    if not os.path.isdir(cifar10_c_folder):
        raise FileNotFoundError(f"CIFAR-10-C not found at {cifar10_c_folder}: unpack "
                                "https://zenodo.org/record/2535967/files/CIFAR-10-C.tar there")
    all_corruptions = []
    labels = None
    for file in sorted(os.listdir(cifar10_c_folder)):
        if file == "labels.npy":
            labels = np.load(os.path.join(cifar10_c_folder, file))
        elif file.endswith(".npy"):
            all_corruptions.append(np.load(os.path.join(cifar10_c_folder, file)))
    num_corruptions = len(all_corruptions)
    all_corruptions = np.concatenate(all_corruptions, axis=0)
    indexes = np.random.default_rng(0).permutation(len(all_corruptions))[:10000]
    images = all_corruptions[indexes]
    labels = np.tile(labels, num_corruptions)[indexes]
    os.makedirs(datasets_folder, exist_ok=True)
    np.save(out[0], images)
    np.save(out[1], labels)


def load_datasets(nominal, datasets_folder: str):
    """`_load_datasets` (case_study_cifar10.py:139-154).  nominal as `cifar10.load_data()` returns it (uint8
    [N, 32, 32, 3], labels [N, 1]); the nominal images become float64 (`x / 255.0`), and so does the OOD set."""
    (x_train, y_train), (x_test, y_test) = nominal
    x_train, x_test = x_train / 255.0, x_test / 255.0
    y_test, y_train = y_test.flatten(), y_train.flatten()
    ood_x_test = np.load(os.path.join(datasets_folder, OOD_FILES[0])).astype("float32") / 255.0
    ood_y_test = np.load(os.path.join(datasets_folder, OOD_FILES[1]))

    ood_x_test = np.concatenate((x_test, ood_x_test), axis=0)
    ood_y_test = np.concatenate((y_test.flatten(), ood_y_test), axis=0)
    shuffle_args = np.random.default_rng(0).permutation(len(ood_y_test))
    return (x_train, y_train), (x_test, y_test), (ood_x_test[shuffle_args], ood_y_test[shuffle_args])


class Cifar10CaseStudy(CaseStudy):
    name = NAME
    num_classes = 10
    batch_size = CIFAR_10_BATCH_SIZE
    epochs = 20
    sa_layers = SA_ACTIVATION_LAYERS
    nc_layers = NC_ACTIVATION_LAYERS
    num_selected = 1000
    prediction_badge_size = CIFAR_10_BATCH_SIZE
    network = staticmethod(network)
