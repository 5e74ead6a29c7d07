"""keras_preprocessing 1.1.2's text_to_word_sequence, Tokenizer (fit_on_texts, texts_to_sequences) and
pad_sequences, restated literally as their Python loops (TEST INFRASTRUCTURE ONLY: Keras cannot be installed
offline).  tests/test_keras_text_oracle.py pins them to known Keras behaviour.

Also: `imdb_like_texts`, seeded synthetic IMDB-like reviews (Zipf words, capitals, punctuation, "<br />"), and
`imdb_inputs`, the case study's recipe (case_study_imdb.py:316-336) with this tokenizer.
"""
from __future__ import annotations

from collections import OrderedDict, defaultdict

import numpy as np

DEFAULT_FILTERS = '!"#$%&()*+,-./:;<=>?@[\\]^_`{|}~\t\n'


def text_to_word_sequence(text, filters=DEFAULT_FILTERS, lower=True, split=" "):
    if lower:
        text = text.lower()
    translate_dict = {c: split for c in filters}
    translate_map = str.maketrans(translate_dict)
    text = text.translate(translate_map)
    seq = text.split(split)
    return [i for i in seq if i]


class Tokenizer(object):
    def __init__(self, num_words=None, filters=DEFAULT_FILTERS, lower=True, split=" ", document_count=0):
        self.word_counts = OrderedDict()
        self.word_docs = defaultdict(int)
        self.filters = filters
        self.split = split
        self.lower = lower
        self.num_words = num_words
        self.document_count = document_count
        self.index_docs = defaultdict(int)
        self.word_index = {}
        self.index_word = {}

    def fit_on_texts(self, texts):
        for text in texts:
            self.document_count += 1
            seq = text_to_word_sequence(text, self.filters, self.lower, self.split)
            for w in seq:
                if w in self.word_counts:
                    self.word_counts[w] += 1
                else:
                    self.word_counts[w] = 1
            for w in set(seq):
                self.word_docs[w] += 1

        wcounts = list(self.word_counts.items())
        wcounts.sort(key=lambda x: x[1], reverse=True)
        sorted_voc = []
        sorted_voc.extend(wc[0] for wc in wcounts)
        self.word_index = dict(zip(sorted_voc, list(range(1, len(sorted_voc) + 1))))
        self.index_word = {c: w for w, c in self.word_index.items()}
        for w, c in list(self.word_docs.items()):
            self.index_docs[self.word_index[w]] = c

    def texts_to_sequences(self, texts):
        return list(self.texts_to_sequences_generator(texts))

    def texts_to_sequences_generator(self, texts):
        num_words = self.num_words
        for text in texts:
            seq = text_to_word_sequence(text, self.filters, self.lower, self.split)
            vect = []
            for w in seq:
                i = self.word_index.get(w)
                if i is not None:
                    if num_words and i >= num_words:
                        continue
                    else:
                        vect.append(i)
            yield vect


def pad_sequences(sequences, maxlen=None, dtype="int32", padding="pre", truncating="pre", value=0.0):
    num_samples = len(sequences)
    lengths = []
    sample_shape = ()
    flag = True
    for x in sequences:
        lengths.append(len(x))
        if flag and len(x):
            sample_shape = np.asarray(x).shape[1:]
            flag = False
    if maxlen is None:
        maxlen = np.max(lengths)
    x = np.full((num_samples, maxlen) + sample_shape, value, dtype=dtype)
    for idx, s in enumerate(sequences):
        if not len(s):
            continue
        if truncating == "pre":
            trunc = s[-maxlen:]
        elif truncating == "post":
            trunc = s[:maxlen]
        else:
            raise ValueError('Truncating type "%s" not understood' % truncating)
        trunc = np.asarray(trunc, dtype=dtype)
        if padding == "post":
            x[idx, :len(trunc)] = trunc
        elif padding == "pre":
            x[idx, -len(trunc):] = trunc
        else:
            raise ValueError('Padding type "%s" not understood' % padding)
    return x


def imdb_inputs(train_texts, test_texts, corrupted_texts, vocab_size=2000, maxlen=100):
    """x_train, x_test, x_corrupted as case_study_imdb.py:321-336 computes them."""
    tokenizer = Tokenizer(num_words=vocab_size)
    tokenizer.fit_on_texts(train_texts)
    return tuple(pad_sequences(tokenizer.texts_to_sequences(t), maxlen=maxlen)
                 for t in (train_texts, test_texts, corrupted_texts))


_PUNCT = [",", ".", "!", "?", "...", "(", ")", "\"", ":", ";", "-", "'s", "<br /><br />"]


def imdb_like_texts(n_texts: int, seed: int, vocab_size: int = 60000, mean_words: int = 230):
    """Seeded reviews of ~mean_words words: Zipf(1.1) draws over vocab_size synthetic words, 8 % capitalised,
    punctuation attached or standing alone, "<br />" line breaks."""
    rng = np.random.default_rng(seed)
    letters = np.array(list("etaoinshrdlcumwfgypbvkjxqz"))
    lens = np.clip(rng.poisson(4.5, size=vocab_size) + 1, 1, 18)
    vocab = ["".join(rng.choice(letters, size=k)) for k in lens]
    p = 1.0 / np.arange(1, vocab_size + 1) ** 1.1
    p /= p.sum()
    texts = []
    for _ in range(n_texts):
        n = max(1, int(rng.normal(mean_words, mean_words / 3)))
        ids = rng.choice(vocab_size, size=n, p=p)
        caps = rng.random(n) < 0.08
        punct = rng.random(n)
        toks = []
        for k, w_id in enumerate(ids):
            w = vocab[w_id]
            if caps[k]:
                w = w.capitalize()
            if punct[k] < 0.1:
                w += _PUNCT[int(punct[k] * 10 * len(_PUNCT)) % len(_PUNCT)]
            toks.append(w)
        texts.append(" ".join(toks))
    return texts
