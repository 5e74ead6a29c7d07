"""CPU tests of the restatement behind the device backend of TextCorruptor.corrupt (oracle/corrupt_oracle.py):
NumPy's SeedSequence -> PCG64 draws, Generator.shuffle / choice and the md5-mod hashes, then corrupt() rebuilt on
those draws alone against the host port, and the tip_corrupt_* argument checks, which run without a device."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from oracle import corrupt_oracle as O
from oracle import text_corruptor_oracle as TO
from simple_tip_b200 import _lib
from simple_tip_b200.core import text_corruptor as T

SEEDS = [0, 1, 2, 7, 999_999, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 40, 2 ** 62 + 12345, 2 ** 63 - 1]


def test_random_equals_numpy():
    rng = np.random.default_rng(0)
    seeds = SEEDS + [int(s) for s in rng.integers(0, 2 ** 63 - 1, size=200)] + list(range(100, 1100, 7))
    for s in seeds:
        want = np.random.default_rng(s).random(1000).tolist()
        r = O.PCG64(s)
        assert [r.random() for _ in range(1000)] == want, s


def test_shuffle_equals_numpy():
    ns = list(range(0, 301)) + [511, 512, 513, 1023, 1024, 1025, 4095, 4097, 65535, 65537]
    for s in SEEDS[:8] + [123456]:
        for n in ns:
            a = np.arange(n)
            np.random.default_rng(s).shuffle(a)
            b = list(range(n))
            O.PCG64(s).shuffle(b)
            assert a.tolist() == b, (s, n)


def test_choice_equals_numpy():
    rng = np.random.default_rng(1)
    for s in SEEDS + list(range(2000, 3000)):
        k = int(rng.integers(1, 6))
        d = 1 / rng.integers(1, 9, size=k).astype(np.float64)
        p = d / d.sum()
        a = np.arange(10, 10 + k)
        assert O.choice(O.PCG64(s), a.tolist(), p) == np.random.default_rng(s).choice(a, p=p), s
    for p in ([0.05, 0.3, 0.3, 0.35], [0.0, 0.5, 0.0, 0.5], [0.0, 0.0, 1.0, 0.0]):
        p = np.array(p) / np.sum(p)
        for s in range(300):
            assert O.choice(O.PCG64(s), [0, 1, 2, 3], p) == np.random.default_rng(s).choice(4, p=p)
    with pytest.raises(ValueError):
        O.choice(O.PCG64(0), [], [])


def test_md5_mod_over_one_to_three_blocks():
    rng = np.random.default_rng(2)
    for n in range(0, 201):
        msg = bytes(rng.integers(0, 256, size=n, dtype=np.uint8))
        assert O.md5_mod(msg) == int(hashlib.md5(msg).hexdigest(), 16) % 10 ** 6
        assert O.md5_mod(msg) == T._hash_text_to_int([msg.decode("latin-1")]) or not msg.isascii()
    assert O.md5_mod(b"kitten 12") == T._hash_text_to_int(["kitten", "12"])


UNICODE_TEXTS = [
    "", "a", "I", "x y", "  leading and trailing  ", "The Movie was GREAT<br /><br />really!!! ...",
    "café naïve résumé über crème brûlée", "café combining accents é̀", "日本語のテキスト 映画 です",
    "emoji 😀😀 party 🎉x", "½ ¾ 3½ 42 1999 2nd", "snake_case __init__ x_y_z", "Éclair ÉCLAIR éclair",
    "ωmega ÿes ñandu ßtrasse", "tab\tnew\nline nbsp em", "a" * 70 + " " + "é" * 40 + " " + "𝔘" * 30,
]


@pytest.fixture(scope="module")
def port(tmp_path_factory):
    """The host port on the golden corpus (its distances from the golden file: no device needed)."""
    g = np.load(TO.GOLDEN, allow_pickle=False)
    corpus = TO.golden_value(g, "corpus")
    tmp = str(tmp_path_factory.mktemp("port"))
    d = os.path.join(tmp, T._hash_text_to_str(list(corpus) + ["250"]))
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, "distances.npy"), g["small_distances"])
    return T.TextCorruptor(corpus, cache_dir=tmp, dictionary_size=250, thesaurus_path=TO.THESAURUS_FIXTURE), corpus


@pytest.mark.parametrize("severity,seed", [(0.0, 0), (0.3, 1), (0.5, 0), (1.0, 2 ** 40)])
def test_corrupt_rebuilt_on_the_restated_draws_equals_the_host_port(port, severity, seed):
    tc, corpus = port
    unicode_texts = UNICODE_TEXTS + [" ".join(tc.common_words[::7]), " ".join(w.upper() for w in tc.common_words[:40])]
    for texts in (corpus, unicode_texts):
        want = tc.corrupt(texts, severity, seed, force_recalculate=True)
        assert O.corrupt(tc, texts, severity, seed) == want
    w = T.CorruptionWeights(0.0, 0.5, 0.0, 0.5)
    assert O.corrupt(tc, corpus, severity, seed, w) == tc.corrupt(corpus, severity, seed, weights=w,
                                                                  force_recalculate=True)


def test_c_abi_checks_the_corrupt_arguments_before_any_launch():
    """Zero texts / words / keys return after the checks, so this runs without a device."""
    lib = _lib.load()
    cdf = (C.c_double * 4)(0.25, 0.5, 0.75, 1.0)
    empty = _lib.CorruptTable()
    ref = C.addressof(empty)
    assert lib.tip_corrupt_table_build(ref, None) == 0
    assert lib.tip_corrupt_count(None, None, 0, None, None, None) == 0
    assert lib.tip_corrupt_texts(None, None, 0, None, None, 0, 0.5, cdf, *([None] * 7), None) == 0
    assert lib.tip_corrupt_texts(None, None, 0, None, None, -1, 0.5, cdf, *([None] * 7), None) != 0   # seed < 0
    assert lib.tip_corrupt_texts(None, None, 0, None, None, 0, 1.5, cdf, *([None] * 7), None) != 0    # severity
    assert lib.tip_corrupt_texts(None, None, -1, None, None, 0, 0.5, cdf, *([None] * 7), None) != 0
    assert lib.tip_corrupt_layout(None, 0, None, None, None, None, None) == 0
    assert lib.tip_corrupt_write(None, None, None, 0, ref, ref, ref, *([None] * 7), None) == 0
    assert lib.tip_corrupt_census(None, 0, None, None) != 0                                          # no bitmap
    bad = _lib.CorruptTable(n=3, cap=4)                                                              # cap < 2 n, nulls
    assert lib.tip_corrupt_table_build(C.addressof(bad), None) != 0
    assert lib.tip_corrupt_write(None, None, None, 0, C.addressof(bad), ref, ref, *([None] * 7), None) != 0
    assert C.sizeof(_lib.CorruptTable) == 88           # nine pointers, two int64


def test_backend_switch_reads_the_environment(monkeypatch):
    monkeypatch.delenv("B200TIP_CORRUPT", raising=False)
    assert T._corrupt_backend(None) == "host"
    monkeypatch.setenv("B200TIP_CORRUPT", "device")
    assert T._corrupt_backend(None) == "device" and T._corrupt_backend("host") == "host"
    with pytest.raises(ValueError):
        T._corrupt_backend("gpu")
