"""keras_preprocessing 1.1.2's word `Tokenizer` and `pad_sequences` (what `tf.keras.preprocessing` runs under
TensorFlow 2.6.1), as the IMDB case study uses them (case_study_imdb.py:321-336), without TensorFlow.

`Tokenizer` splits, counts and looks words up on the GPU (csrc/tokenizer.cu): its `word_counts`, `word_index`,
`index_word` and `document_count` equal Keras', including order, and its sequences are Keras' lists.  `word_docs`
and `index_docs` hold Keras' values, in first-occurrence order: Keras fills them from `set(seq)`, whose order
follows PYTHONHASHSEED.  `texts_to_padded` fuses `texts_to_sequences` and `pad_sequences` on the device.
`pad_sequences` is the host function, for callers who already hold sequences.
"""
from __future__ import annotations

from collections import OrderedDict, defaultdict
from typing import List, Optional, Sequence

import numpy as np

DEFAULT_FILTERS = '!"#$%&()*+,-./:;<=>?@[\\]^_`{|}~\t\n'


def _check_texts(texts) -> List[str]:
    texts = list(texts)
    for t in texts:
        if not isinstance(t, str):
            raise TypeError(f"texts must be str, got {type(t).__name__}: pre-tokenised (list) texts are not supported")
    return texts


def _check_padding(padding: str, truncating: str) -> None:
    if truncating not in ("pre", "post"):
        raise ValueError('Truncating type "%s" not understood' % truncating)
    if padding not in ("pre", "post"):
        raise ValueError('Padding type "%s" not understood' % padding)


class Tokenizer(object):
    """keras_preprocessing.text.Tokenizer with the default word analyzer.  Not supported (NotImplementedError):
    `char_level`, `analyzer`, `oov_token`, a `split` other than one ASCII character, non-ASCII `filters`."""

    def __init__(self, num_words: Optional[int] = None, filters: str = DEFAULT_FILTERS, lower: bool = True,
                 split: str = " ", char_level: bool = False, oov_token=None, document_count: int = 0,
                 analyzer=None):
        if char_level:
            raise NotImplementedError("char_level tokenization is not supported")
        if analyzer is not None:
            raise NotImplementedError("a custom analyzer is not supported")
        if oov_token is not None:
            raise NotImplementedError("oov_token is not supported")
        if not isinstance(split, str) or len(split) != 1 or not split.isascii():
            raise NotImplementedError("split must be one ASCII character")
        if not filters.isascii():
            raise NotImplementedError("filters must be ASCII characters")
        self.word_counts = OrderedDict()
        self.word_docs = defaultdict(int)
        self.filters = filters
        self.split = split
        self.lower = lower
        self.num_words = num_words
        self.document_count = document_count
        self.char_level = char_level
        self.oov_token = oov_token
        self.index_docs = defaultdict(int)
        self.word_index = {}
        self.index_word = {}
        self.analyzer = analyzer
        self._hash_bits = 64        # word-table hash width; tests narrow it to force collisions
        self._arena = bytearray()   # the vocabulary's (lowered) bytes, in word_counts order
        self._vstart: List[int] = []
        self._vlen: List[int] = []
        self._counts = np.zeros(0, dtype=np.int64)
        self._v_index = np.zeros(0, dtype=np.int32)
        self._vocab = None          # engine.TokVocab of the current vocabulary, built on first use

    def _separators(self):
        from .. import engine as E

        return E.separator_mask(self.filters + self.split)

    def _device_vocab(self):
        from .. import engine as E

        if self._vocab is None or self._vocab.hash_bits != self._hash_bits:
            self._vocab = E.TokVocab(bytes(self._arena), np.asarray(self._vstart, dtype=np.int64),
                                     np.asarray(self._vlen, dtype=np.int32), self._v_index, self._hash_bits)
        return self._vocab

    def _words(self, texts: List[str]):
        from .. import engine as E

        raw, off = E.encode_texts(texts, self.lower)
        return raw, E.TokWords(raw, off, self._separators(), self.lower, self._hash_bits)

    def fit_on_texts(self, texts: Sequence[str]) -> None:
        texts = _check_texts(texts)
        self.document_count += len(texts)
        if texts:
            from .. import engine as E

            raw, words = self._words(texts)
            if words.n_words:
                self._add_counts(raw, E.tok_fit(words, self._device_vocab()))
        rank = np.argsort(-self._counts, kind="stable")          # list.sort(key=count, reverse=True) is stable
        vocab = list(self.word_counts)
        sorted_voc = [vocab[i] for i in rank]
        self.word_index = dict(zip(sorted_voc, range(1, len(sorted_voc) + 1)))
        self.index_word = {c: w for w, c in self.word_index.items()}
        for w, c in self.word_docs.items():
            self.index_docs[self.word_index[w]] = c
        self._v_index = np.empty(len(rank), dtype=np.int32)
        self._v_index[rank] = np.arange(1, len(rank) + 1, dtype=np.int32)
        self._vocab = None

    def _add_counts(self, raw: bytes, cols: np.ndarray) -> None:
        """Merges tok_fit's columns (by first occurrence: the old vocabulary's entries, then new words) into
        word_counts / word_docs and the device vocabulary's bytes."""
        nv = len(self._vstart)
        first, count, docs, start, length = cols
        old = first < nv
        vocab = list(self.word_counts) if old.any() else []
        for i, c, d in zip(first[old].tolist(), count[old].tolist(), docs[old].tolist()):
            self.word_counts[vocab[i]] += c
            self.word_docs[vocab[i]] += d
        new_counts = count[~old]
        for s, n, c, d in zip(start[~old].tolist(), length[~old].tolist(), new_counts.tolist(), docs[~old].tolist()):
            b = raw[s:s + n]
            if self.lower:
                b = b.lower()                                   # the ASCII lowering the device did in place
            w = b.decode("utf-8", "surrogatepass")
            self.word_counts[w] = c
            self.word_docs[w] = d
            self._vstart.append(len(self._arena))
            self._vlen.append(n)
            self._arena += b
        counts = np.zeros(nv + len(new_counts), dtype=np.int64)
        counts[:nv] = self._counts
        np.add.at(counts, first[old], count[old])
        counts[nv:] = new_counts
        self._counts = counts

    def _lookup(self, texts: List[str], ragged: bool, maxlen=None, padding="pre", truncating="pre", value=0):
        from .. import engine as E

        _, words = self._words(texts)
        return E.tok_lookup(words, self._device_vocab(), self.num_words or 0, ragged, maxlen, padding,
                            truncating, value)

    def texts_to_sequences(self, texts: Sequence[str]) -> List[List[int]]:
        """Keras' lists of word indexes; unknown words and indexes >= num_words are dropped."""
        texts = _check_texts(texts)
        if not texts:
            return []
        ids, kept_off, _ = self._lookup(texts, ragged=True)
        off = kept_off.cpu().numpy()
        ids = ids[:int(off[-1])].cpu().numpy()
        return [ids[off[i]:off[i + 1]].tolist() for i in range(len(texts))]

    def texts_to_padded(self, texts: Sequence[str], maxlen: int, padding: str = "pre", truncating: str = "pre",
                        value: int = 0, device_out: bool = False):
        """pad_sequences(self.texts_to_sequences(texts), maxlen, dtype="int32", padding, truncating, value) in one
        device pass: int32 [len(texts), maxlen], a NumPy array or, with device_out, a CUDA tensor."""
        import torch

        texts = _check_texts(texts)
        if isinstance(maxlen, bool) or not isinstance(maxlen, (int, np.integer)) or maxlen < 1:
            raise ValueError(f"maxlen must be a positive int, got {maxlen!r}")
        _check_padding(padding, truncating)
        if int(value) != value or not -2 ** 31 <= int(value) < 2 ** 31:
            raise ValueError(f"value must be an int32, got {value!r}")
        if not texts:
            out = torch.empty((0, int(maxlen)), dtype=torch.int32)
            if device_out:
                from .. import engine as E

                out = out.to(E.require_cuda())
            return out if device_out else out.numpy()
        _, _, padded = self._lookup(texts, False, int(maxlen), padding, truncating, int(value))
        return padded if device_out else padded.cpu().numpy()


def pad_sequences(sequences, maxlen=None, dtype="int32", padding="pre", truncating="pre", value=0.0):
    """keras_preprocessing.sequence.pad_sequences 1.1.2, on the host."""
    if not hasattr(sequences, "__len__"):
        raise ValueError("`sequences` must be iterable.")
    num_samples = len(sequences)
    lengths = []
    sample_shape = ()
    flag = True
    for x in sequences:
        try:
            lengths.append(len(x))
            if flag and len(x):
                sample_shape = np.asarray(x).shape[1:]
                flag = False
        except TypeError:
            raise ValueError("`sequences` must be a list of iterables. Found non-iterable: " + str(x))
    if maxlen is None:
        maxlen = np.max(lengths)
    is_dtype_str = np.issubdtype(dtype, np.str_)
    if isinstance(value, str) and dtype != object and not is_dtype_str:
        raise ValueError("`dtype` {} is not compatible with `value`'s type: {}\n"
                         "You should set `dtype=object` for variable length strings.".format(dtype, type(value)))
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
        if trunc.shape[1:] != sample_shape:
            raise ValueError("Shape of sample %s of sequence at position %s is different from expected shape %s"
                             % (trunc.shape[1:], idx, sample_shape))
        if padding == "post":
            x[idx, :len(trunc)] = trunc
        elif padding == "pre":
            x[idx, -len(trunc):] = trunc
        else:
            raise ValueError('Padding type "%s" not understood' % padding)
    return x
