"""CPU tests: the keras_preprocessing 1.1.2 restatement of oracle/keras_text_oracle.py against known Keras
behaviour, the host pad_sequences against it, the Tokenizer's unsupported options, and load_datasets."""
import numpy as np
import pytest

from oracle import keras_text_oracle as K
from simple_tip_b200.core import imdb
from simple_tip_b200.core.tokenizer import Tokenizer, pad_sequences


def test_word_sequence_keeps_apostrophes_and_splits_only_on_filters_and_space():
    assert K.text_to_word_sequence("Don't STOP, it's fine!") == ["don't", "stop", "it's", "fine"]
    assert K.text_to_word_sequence("a\tb\nc") == ["a", "b", "c"]
    # \r, no-break space and the line separator are neither filters nor the split character
    assert K.text_to_word_sequence("a\rb c\xa0d e\u2028f") == ["a\rb", "c\xa0d", "e\u2028f"]
    assert K.text_to_word_sequence("  ,,  ") == []
    assert K.text_to_word_sequence("A-B", lower=False) == ["A", "B"]
    assert K.text_to_word_sequence("x|y|z", filters="", split="|") == ["x", "y", "z"]


def test_fit_orders_ties_by_first_occurrence_and_counts_documents():
    tok = K.Tokenizer()
    tok.fit_on_texts(["b a c", "c b b", "d"])
    assert list(tok.word_counts.items()) == [("b", 3), ("a", 1), ("c", 2), ("d", 1)]
    assert tok.word_index == {"b": 1, "c": 2, "a": 3, "d": 4}
    assert dict(tok.word_docs) == {"b": 2, "a": 1, "c": 2, "d": 1}
    assert dict(tok.index_docs) == {1: 2, 3: 1, 2: 2, 4: 1}
    assert tok.document_count == 3
    tok.fit_on_texts(["d d d e"])                     # a second fit accumulates
    assert tok.word_index == {"d": 1, "b": 2, "c": 3, "a": 4, "e": 5} and tok.document_count == 4


def test_num_words_keeps_indices_below_it():
    tok = K.Tokenizer(num_words=3)
    tok.fit_on_texts(["a a a b b c"])
    assert tok.texts_to_sequences(["c b a zzz a"]) == [[2, 1, 1]]
    for n, want in ((None, [[3, 2, 1]]), (0, [[3, 2, 1]]), (1, [[]]), (2, [[1]])):
        tok.num_words = n
        assert tok.texts_to_sequences(["c b a"]) == want


def test_pre_truncation_keeps_the_last_tokens_and_empty_texts_give_zero_rows():
    x = K.pad_sequences([[1, 2, 3, 4], [], [5]], maxlen=3)
    assert x.dtype == np.int32 and x.tolist() == [[2, 3, 4], [0, 0, 0], [0, 0, 5]]
    assert K.pad_sequences([[1, 2, 3, 4]], maxlen=3, truncating="post", padding="post").tolist() == [[1, 2, 3]]
    assert K.pad_sequences([[1], [2, 3]], maxlen=3, padding="post", value=-7).tolist() == [[1, -7, -7], [2, 3, -7]]


@pytest.mark.parametrize("padding", ["pre", "post"])
@pytest.mark.parametrize("truncating", ["pre", "post"])
def test_host_pad_sequences_equals_the_restatement(padding, truncating):
    rng = np.random.default_rng(0)
    seqs = [rng.integers(1, 50, size=int(k)).tolist() for k in rng.integers(0, 12, size=200)]
    for maxlen in (None, 1, 5, 11, 30):
        for value in (0, -1, 7):
            got = pad_sequences(seqs, maxlen=maxlen, padding=padding, truncating=truncating, value=value)
            want = K.pad_sequences(seqs, maxlen=maxlen, padding=padding, truncating=truncating, value=value)
            assert got.dtype == want.dtype and np.array_equal(got, want)
    with pytest.raises(ValueError, match="not understood"):
        pad_sequences(seqs, maxlen=3, padding="middle")


@pytest.mark.parametrize("kwargs", [dict(char_level=True), dict(analyzer=str.split), dict(oov_token="<oov>"),
                                    dict(split="ab"), dict(split="\xa0"), dict(filters="!—")])
def test_unsupported_tokenizer_options_raise(kwargs):
    with pytest.raises(NotImplementedError):
        Tokenizer(**kwargs)


def test_non_str_texts_raise_type_error_before_the_device():
    tok = Tokenizer()
    with pytest.raises(TypeError):
        tok.fit_on_texts([["already", "split"]])
    with pytest.raises(TypeError):
        tok.texts_to_sequences(["fine", b"bytes"])
    with pytest.raises(ValueError, match="maxlen"):
        tok.texts_to_padded(["a"], maxlen=0)
    with pytest.raises(ValueError, match="not understood"):
        tok.texts_to_padded(["a"], maxlen=3, truncating="middle")


def test_load_datasets_concatenates_and_shuffles_with_the_global_rng(tmp_path):
    rng = np.random.default_rng(1)
    x_train, x_test, x_corr = (rng.integers(0, 2000, size=(n, 100)).astype(np.int32) for n in (7, 5, 5))
    y_train, y_test = [0, 1, 1, 0, 1, 0, 0], [1, 0, 1, 1, 0]
    for name, a in zip(imdb.FILES, (x_train, y_train, x_test, y_test, x_corr)):
        np.save(tmp_path / name, a)
    np.random.seed(3)
    (a, b), (c, d), (e, f) = imdb.load_datasets(str(tmp_path))
    np.random.seed(3)
    perm = np.random.permutation(10)
    assert np.array_equal(a, x_train) and b.tolist() == y_train and np.array_equal(c, x_test) and d.tolist() == y_test
    assert np.array_equal(e, np.concatenate([x_test, x_corr])[perm]) and f.tolist() == np.array(y_test * 2)[perm].tolist()
    (_, _), (_, _), (e2, _) = imdb.load_datasets(str(tmp_path), rng=np.random.default_rng(5))
    assert np.array_equal(e2, np.concatenate([x_test, x_corr])[np.random.default_rng(5).permutation(10)])


def test_prepare_datasets_returns_early_when_the_files_exist(tmp_path):
    for name in imdb.FILES:
        np.save(tmp_path / name, np.zeros(1))
    imdb.prepare_datasets(str(tmp_path), ["never", "read"], [0, 1], [1], [0])   # no corruptor, no device
    assert sorted(p.name for p in tmp_path.iterdir()) == sorted(imdb.FILES)
