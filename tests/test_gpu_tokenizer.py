"""GPU tests of the device tokenizer (csrc/tokenizer.cu, core/tokenizer.py) against the keras_preprocessing 1.1.2
restatement of oracle/keras_text_oracle.py, exactly, and of core.imdb.prepare_datasets end to end."""
import io
import itertools

import numpy as np
import pytest

from oracle import keras_text_oracle as K
from oracle import text_corruptor_oracle as TO
from simple_tip_b200 import _lib
from simple_tip_b200.core import imdb
from simple_tip_b200.core.text_corruptor import TextCorruptor
from simple_tip_b200.core.tokenizer import Tokenizer

pytestmark = pytest.mark.gpu

PADS = list(itertools.product(("pre", "post"), ("pre", "post")))


def _golden_corpus():
    return TO.golden_value(np.load(TO.GOLDEN), "corpus")


def _synthetic(n, seed):
    return TO.synthetic_corpus(TO.thesaurus_headwords(TO.THESAURUS_FIXTURE, 300, seed=seed), n, seed=seed + 1)


def _adversarial():
    rng = np.random.default_rng(5)
    texts = ["", " ", ",,, !!  ", "\t\n", "a", "A", "Don't STOP, it's fine!", "a\rb c\xa0d e\u2028f",
             "İstanbul İ İİ", "ΟΔΟΣ ΟΔΟΣ. Σ ΣΑΣ σας", "\ud800 abc\udfff 😀 😀 \udfff\ud800",
             "x" * 100_000, "y " + "x" * 100_000 + " z", "<br /><br />Br BR"]
    for k in (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257):
        texts.append("b" * k)
        texts.append("".join(rng.choice(list("ab ,.C"), size=k)))
        texts.append(" " * (k - 1) + "q")
    words = ["w%d" % i for i in range(3000)]
    big = " ".join(words[int(i)] for i in rng.zipf(1.3, size=260_000) % 3000)
    texts.append(big[:1_000_000])                                          # one 1 MB text
    return texts


def _check_fit(tok, ref):
    assert list(tok.word_counts.items()) == list(ref.word_counts.items())
    assert list(tok.word_index.items()) == list(ref.word_index.items())
    assert tok.index_word == ref.index_word
    assert dict(tok.word_docs) == dict(ref.word_docs)
    assert dict(tok.index_docs) == dict(ref.index_docs)
    assert tok.document_count == ref.document_count


def _check_outputs(tok, ref, texts, maxlens=(1, 7, 100), values=(0,)):
    seqs = ref.texts_to_sequences(texts)
    assert tok.texts_to_sequences(texts) == seqs
    for (padding, truncating), maxlen, value in itertools.product(PADS, maxlens, values):
        got = tok.texts_to_padded(texts, maxlen, padding=padding, truncating=truncating, value=value)
        want = K.pad_sequences(seqs, maxlen=maxlen, padding=padding, truncating=truncating, value=value)
        assert got.dtype == np.int32 and want.dtype == np.int32
        assert np.array_equal(got, want), (padding, truncating, maxlen, value)


def _fit_both(texts, hash_bits=64, **kwargs):
    tok, ref = Tokenizer(**kwargs), K.Tokenizer(**kwargs)
    tok._hash_bits = hash_bits
    tok.fit_on_texts(texts)
    ref.fit_on_texts(texts)
    _check_fit(tok, ref)
    return tok, ref


@pytest.mark.parametrize("num_words", [None, 0, 1, 2000])
def test_synthetic_corpus_matches_keras(num_words):
    train, test = _golden_corpus(), _synthetic(150, 3)
    tok, ref = _fit_both(train, num_words=num_words)
    _check_outputs(tok, ref, test + train[:50], values=(0, -5))


def test_adversarial_texts_match_keras():
    texts = _adversarial()
    tok, ref = _fit_both(texts, num_words=50)
    _check_outputs(tok, ref, texts, maxlens=(1, 100, 129))
    tok, ref = _fit_both(texts[:-1], lower=False)
    _check_outputs(tok, ref, texts[:-1], maxlens=(100,))
    tok, ref = _fit_both(texts[:-1], filters="", split="b")
    _check_outputs(tok, ref, texts[:-1], maxlens=(100,))


def test_two_fits_accumulate_as_in_keras():
    a, b = _golden_corpus(), _synthetic(120, 7) + _adversarial()[:20]
    tok, ref = _fit_both(a, num_words=300)
    tok.fit_on_texts(b)
    ref.fit_on_texts(b)
    _check_fit(tok, ref)
    _check_outputs(tok, ref, b + a[:30], maxlens=(100,))
    tok.fit_on_texts([])
    ref.fit_on_texts([])
    _check_fit(tok, ref)


@pytest.mark.parametrize("hash_bits", [1, 3, 12])
def test_narrow_hashes_force_collisions_without_changing_a_result(hash_bits):
    train = _golden_corpus()
    tok, ref = _fit_both(train[:100], hash_bits=hash_bits, num_words=200)
    tok.fit_on_texts(train[100:])
    ref.fit_on_texts(train[100:])
    _check_fit(tok, ref)
    _check_outputs(tok, ref, _synthetic(60, 9) + train[:20], maxlens=(100,))


def test_texts_before_any_fit_give_empty_sequences():
    tok = Tokenizer()
    assert tok.texts_to_sequences(["a b", ""]) == [[], []]
    assert np.array_equal(tok.texts_to_padded(["a b", ""], 4, value=9), np.full((2, 4), 9, np.int32))


def test_device_out_returns_the_padded_rows_on_the_gpu():
    import torch

    train = _golden_corpus()
    tok, ref = _fit_both(train, num_words=2000)
    got = tok.texts_to_padded(train, 100, device_out=True)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.dtype == torch.int32
    assert np.array_equal(got.cpu().numpy(), K.pad_sequences(ref.texts_to_sequences(train), maxlen=100))


def test_empty_inputs_launch_nothing():
    tok = Tokenizer()
    tok.fit_on_texts(["some words here"])
    before = _lib.launch_count()
    tok.fit_on_texts([])
    assert tok.texts_to_sequences([]) == []
    assert tok.texts_to_padded([], 100).shape == (0, 100)
    assert tok.texts_to_padded([], 100, device_out=True).shape == (0, 100)
    assert _lib.launch_count() == before


def _npy_bytes(a) -> bytes:
    f = io.BytesIO()
    np.save(f, a)
    return f.getvalue()


def test_prepare_datasets_writes_the_reference_recipes_files(tmp_path):
    corpus = _golden_corpus()
    train, test = corpus[:120], corpus[120:]
    y_train, y_test = [i % 2 for i in range(len(train))], [(i // 3) % 2 for i in range(len(test))]
    folder = tmp_path / "imdb"
    imdb.prepare_datasets(str(folder), train, y_train, test, y_test, thesaurus_path=TO.THESAURUS_FIXTURE)

    corruptor = TextCorruptor(base_dataset=train + test, cache_dir=str(tmp_path / "ref"),
                              thesaurus_path=TO.THESAURUS_FIXTURE)
    ood = corruptor.corrupt(test, severity=0.5, seed=0)
    x_train, x_test, x_corr = K.imdb_inputs(train, test, ood, imdb.VOCAB_SIZE, imdb.INPUT_MAXLEN)
    for name, want in zip(imdb.FILES, (x_train, y_train, x_test, y_test, x_corr)):
        assert (folder / name).read_bytes() == _npy_bytes(want), name
    mtimes = [(folder / f).stat().st_mtime_ns for f in imdb.FILES]
    imdb.prepare_datasets(str(folder), train, y_train, test, y_test, thesaurus_path=TO.THESAURUS_FIXTURE)
    assert [(folder / f).stat().st_mtime_ns for f in imdb.FILES] == mtimes
