"""The IMDB case study's model inputs (case_study_imdb.py:23-25, 271-344) without TensorFlow: the five .npy files
`ImdbCaseStudy._prefetch_datasets` writes and `_load_datasets` reads back.

Nothing here downloads: the caller supplies the texts and labels (e.g. from a local Hugging Face cache) and a local
thesaurus for IMDB-C.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence

import numpy as np

from .text_corruptor import TextCorruptor
from .tokenizer import Tokenizer

VOCAB_SIZE = 2000
INPUT_MAXLEN = 100
FILES = ("x_train.npy", "y_train.npy", "x_test.npy", "y_test.npy", "x_corrupted.npy")


def prepare_datasets(folder: str, train_texts: Sequence[str], train_labels: Sequence[int], test_texts: Sequence[str],
                     test_labels: Sequence[int], thesaurus_path: Optional[str] = None) -> None:
    """`_prefetch_datasets` (:296-344) into `folder` (the reference's <assets>/.external_datasets/imdb): IMDB-C by
    TextCorruptor(train + test, cache_dir=<folder>/corruptor).corrupt(test, severity=0.5, seed=0), a
    Tokenizer(num_words=VOCAB_SIZE) fitted on the training texts, every set padded to INPUT_MAXLEN (int32), the
    labels saved as np.save stores a list of Python ints.  Returns at once when all five files exist."""
    if all(os.path.exists(os.path.join(folder, f)) for f in FILES):
        return
    train_texts, test_texts = list(train_texts), list(test_texts)
    corruptor = TextCorruptor(base_dataset=train_texts + test_texts, cache_dir=os.path.join(folder, "corruptor"),
                              thesaurus_path=thesaurus_path)
    x_test_ood = corruptor.corrupt(test_texts, severity=0.5, seed=0)

    tokenizer = Tokenizer(num_words=VOCAB_SIZE)
    tokenizer.fit_on_texts(train_texts)
    x_train, x_test, x_corrupted = (tokenizer.texts_to_padded(t, INPUT_MAXLEN)
                                    for t in (train_texts, test_texts, x_test_ood))

    os.makedirs(folder, exist_ok=True)
    arrays = (x_train, [int(v) for v in train_labels], x_test, [int(v) for v in test_labels], x_corrupted)
    for name, a in zip(FILES, arrays):
        np.save(os.path.join(folder, name), a)


def load_datasets(folder: str, rng: Optional[np.random.Generator] = None):
    """`_load_datasets` (:271-285): ((x_train, y_train), (x_test, y_test), (ood_x_test, ood_y_test)), the OOD set
    being the nominal and corrupted test sets concatenated and shuffled by `rng.permutation` (None: NumPy's
    global, unseeded `np.random.permutation`, as the reference)."""
    x_train, y_train, x_test, y_test, corrupted_x_test = (np.load(os.path.join(folder, f)) for f in FILES)
    ood_x_test = np.concatenate((x_test, corrupted_x_test), axis=0)
    ood_y_test = np.concatenate((y_test, y_test), axis=0)
    perm = (np.random if rng is None else rng).permutation(len(ood_x_test))
    return (x_train, y_train), (x_test, y_test), (ood_x_test[perm], ood_y_test[perm])
