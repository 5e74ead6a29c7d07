"""GPU tests of tip_levenshtein (the all-pairs Levenshtein matrix of IMDB-C's dictionary) against the plain DP of
oracle/lev_oracle.c, bit for bit, and of TextCorruptor computing its distances on the device."""
import numpy as np
import pytest

from oracle import text_corruptor_oracle as TO
from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E
from simple_tip_b200.core import text_corruptor as T

pytestmark = pytest.mark.gpu


def _words(rng, n, alphabet, lengths):
    return ["".join(rng.choice(alphabet, size=int(k))) for k in rng.choice(lengths, size=n)]


def _check(a, b=None):
    got = E.levenshtein(a, b).cpu().numpy()
    want = TO.levenshtein_matrix(a, b)
    assert got.dtype == np.uint8 and got.shape == want.shape
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    return got


def test_random_ascii_words_of_every_length():
    rng = np.random.default_rng(0)
    ascii_ = [chr(c) for c in range(32, 127)]
    _check(_words(rng, 300, ascii_, np.arange(0, 256)))
    _check(_words(rng, 200, list("ab"), np.arange(0, 256)))          # many ties and long runs


def test_large_alphabet_with_non_bmp_code_points():
    rng = np.random.default_rng(1)
    alphabet = [chr(c) for c in range(0x400, 0x400 + 900)] + [chr(c) for c in range(0x1F300, 0x1F300 + 200)]
    words = _words(rng, 250, alphabet, np.arange(0, 40))
    words += _words(rng, 50, alphabet[:5] + alphabet[-5:], np.arange(0, 130))   # ids below and above 64 mixed
    _check(words)


def test_lengths_around_the_64_bit_blocks():
    rng = np.random.default_rng(2)
    words = []
    for k in (63, 64, 65, 128, 129, 255):
        base = "".join(rng.choice(list("abcd"), size=k))
        words += [base, base[: k // 2] + "z" + base[k // 2 + 1:], base[::-1]]
    words += ["", "a", "ab", "abcd" * 60, "abcd" * 60, ""]                  # identical words, empty vs long
    d = _check(words)
    assert d[words.index(""), words.index("abcd" * 60)] == 240


def test_rectangular_blocks_and_single_rows():
    rng = np.random.default_rng(3)
    a = _words(rng, 70, list("abcdefgh"), np.arange(0, 90))
    b = _words(rng, 333, list("abcdefghij"), np.arange(0, 90))
    _check(a, b)
    _check(b[:1], a)
    _check(a, b[:1])
    for w in ("", "abc", b[7]):
        got = T._levensthein_distance(w, b)
        assert got.dtype == np.float64 and got.shape == (333,)
        assert np.array_equal(got, TO.levenshtein_matrix([w], b)[0].astype(np.float64))


def test_full_4000_word_matrix_with_imdb_like_lengths():
    rng = np.random.default_rng(4)
    lengths = np.clip(np.round(rng.gamma(6.0, 1.4, size=4000)) + 5, 5, 30).astype(int)   # dictionary words: > 4
    letters = list("etaoinshrdlcumwfgypbvkjxqz")
    p = np.linspace(2.0, 0.1, len(letters))
    words = sorted({"".join(rng.choice(letters, size=k, p=p / p.sum())) for k in lengths})
    d = _check(words)
    assert np.array_equal(d, d.T) and not np.any(np.diag(d))


def test_overlong_word_raises_before_any_launch():
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="word 1 has 256 code points"):
        E.levenshtein(["abc", "x" * 256, "y" * 300])
    assert _lib.launch_count() == before


def test_empty_and_single_word_dictionaries_have_the_reference_shapes(tmp_path):
    assert E.levenshtein([]).shape == (0, 0)
    assert T._levensthein_distance("abc", []).shape == (0,)
    for corpus, shape in ((["tiny cat and dog"], (0,)), (["lonely"], (1, 1))):
        tc = T.TextCorruptor(corpus, cache_dir=str(tmp_path), thesaurus_path=TO.THESAURUS_FIXTURE)
        assert tc.lev_dist.shape == shape and tc.lev_dist.dtype == np.uint8 and not tc.lev_dist.any()


def test_text_corruptor_computes_the_golden_distances_and_corruptions():
    from tests.test_text_corruptor_host import run_golden_check

    res = run_golden_check("device")
    assert res and all(res.values()), [k for k, v in res.items() if not v]
