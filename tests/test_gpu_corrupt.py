"""GPU tests of TextCorruptor.corrupt(backend="device") (csrc/corrupt.cu): string for string the host port's output,
in one process (the synonym lists follow the process's set order), on the golden corpus and on texts built to reach
every branch, its golden corruptions under PYTHONHASHSEED=0, independence of order, subset and chunking, the cache
file, tiny dictionaries and the refused inputs."""
import json
import os
import pickle

import numpy as np
import pytest

from oracle import text_corruptor_oracle as TO
from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E
from simple_tip_b200.core import text_corruptor as T

pytestmark = pytest.mark.gpu

EXTRA_THESAURUS = [
    {"word": "movie", "synonyms": ["motion picture", "film", "moving picture show", "flick"]},
    {"word": "café", "synonyms": ["coffee house", "bistro", "brasserie"]},
    {"word": "great", "synonyms": ["very good", "grand", "ótimo", "大きい"]},
    {"word": "naïve", "synonyms": ["simple", "unsophisticated"]},
    {"word": "lonely", "synonyms": ["alone"]},                          # one synonym: not kept (reference rule)
]

SPECIAL = [
    "", "a", "I", "ok", "x y", "   ", "  leading and trailing  ", "The Movie was GREAT<br /><br />really!!! ...",
    "great movie , great café !!! naïve naïve naïve", "café naïve résumé über crème brûlée façade",
    "combining accents: café naïve ééé", "日本語のテキスト 映画 です 。", "emoji 😀😀 party 🎉x 👍🏽",
    "½ ¾ 3½ 42 1999 2nd 0_0 __init__ snake_case", "Éclair ÉCLAIR éclair Über ÜBER", "ωmega ÿes ñandu ßtrasse Ωmega",
    "tab\tnew\nline nbsp em　ideographic", "éé éa aé ñññ ωω ÿÿÿÿ",
    "a" * 70 + " " + "é" * 40 + " " + "𝔘" * 30 + " " + "pneumonoultramicroscopicsilicovolcanoconiosis" * 3,
]


def _thesaurus(tmp_path):
    path = str(tmp_path / "thesaurus.jsonl")
    with open(TO.THESAURUS_FIXTURE) as f, open(path, "w") as g:
        g.write(f.read())
        for line in EXTRA_THESAURUS:
            g.write(json.dumps(line, ensure_ascii=False) + "\n")
    return path


@pytest.fixture(scope="module")
def corpus():
    return TO.golden_value(np.load(TO.GOLDEN, allow_pickle=False), "corpus")


@pytest.fixture(scope="module")
def texts(corpus):
    rng = np.random.default_rng(3)
    big = " ".join(corpus[int(k)] for k in rng.integers(0, len(corpus), size=400))     # > 64 KB
    assert len(big.encode()) > 65536
    return list(corpus[:80]) + SPECIAL + [big] + [" ".join(SPECIAL)]


@pytest.fixture(scope="module")
def tc(tmp_path_factory, corpus):
    tmp = tmp_path_factory.mktemp("tc")
    base = list(corpus) + SPECIAL
    return T.TextCorruptor(base, cache_dir=None, dictionary_size=400, thesaurus_path=_thesaurus(tmp))


@pytest.mark.parametrize("severity", [0.0, 0.3, 0.5, 1.0])
@pytest.mark.parametrize("seed", [0, 1, 2 ** 40])
def test_device_equals_host_string_for_string(tc, texts, severity, seed):
    for w in (None, T.CorruptionWeights(0.0, 0.5, 0.5, 0.0), T.CorruptionWeights(1.0, 0.0, 0.0, 0.0),
              T.CorruptionWeights(0.0, 0.0, 0.0, 1.0)):
        want = tc.corrupt(texts, severity, seed, weights=w, backend="host")
        got = tc.corrupt(texts, severity, seed, weights=w, backend="device")
        assert len(got) == len(want)
        bad = [k for k, (a, b) in enumerate(zip(got, want)) if a != b]
        assert not bad, (bad[:3], [got[k][:200] for k in bad[:2]], [want[k][:200] for k in bad[:2]])


def test_typos_at_non_ascii_letters_and_every_type_are_reached(tc, texts):
    """Severity 1 with typo weight 1: every word of >= 2 code points is a typo, many of them at a non-ASCII
    code point (the replacement changes the UTF-8 length)."""
    words = [w for t in SPECIAL for w in T.split_by_whitespace([t])[0] if len(w) >= 2 and not w.isascii()]
    hit = [w for w in words for s in range(50) if not w[s % len(w)].isascii()]
    assert hit
    w = T.CorruptionWeights(1.0, 0.0, 0.0, 0.0)
    assert tc.corrupt(SPECIAL, 1.0, 0, weights=w, backend="device") == tc.corrupt(SPECIAL, 1.0, 0, weights=w,
                                                                                   backend="host")
    out = tc.corrupt(["great movie café"] * 40, 1.0, 7, weights=T.CorruptionWeights(0, 0, 0, 1), backend="device")
    assert any(" " in s.replace("great movie café", "") for s in out)     # multi-word synonyms came out


def test_golden_corruptions_with_the_device_backend(monkeypatch):
    from tests.test_text_corruptor_host import run_golden_check

    monkeypatch.setenv("B200TIP_CORRUPT", "device")
    res = run_golden_check("cached")
    assert res and all(res.values()), [k for k, v in res.items() if not v]


def test_order_subset_and_chunking_do_not_change_a_text(tc, texts):
    want = tc.corrupt(texts, 0.5, 3, backend="device")
    perm = np.random.default_rng(0).permutation(len(texts))
    assert tc.corrupt([texts[k] for k in perm], 0.5, 3, backend="device") == [want[k] for k in perm]
    sub = perm[: len(perm) // 3]
    assert tc.corrupt([texts[k] for k in sub], 0.5, 3, backend="device") == [want[k] for k in sub]
    cdf = np.array([0.05, 0.35, 0.65, 1.0])
    enc = [t.encode() for t in texts]
    full, bad = E.corrupt_texts(enc, tc.device_tables(), 3, 0.5, cdf)
    assert bad is None
    for chunk in (1, 100, 5000, 70000):
        got, bad = E.corrupt_texts(enc, tc.device_tables(), 3, 0.5, cdf, chunk_bytes=chunk)
        assert bad is None and got == full, chunk


def test_the_device_cache_file_is_the_host_cache_file(tmp_path, corpus):
    th = _thesaurus(tmp_path)
    pickles = {}
    for backend in ("host", "device"):
        d = str(tmp_path / backend)
        tc = T.TextCorruptor(list(corpus), cache_dir=d, dictionary_size=250, thesaurus_path=th)
        out = tc.corrupt(list(corpus), 0.5, 1, backend=backend)
        (f,) = os.listdir(os.path.join(tc.cache_dir, "corrupted"))
        with open(os.path.join(tc.cache_dir, "corrupted", f), "rb") as g:
            pickles[backend] = g.read()
        assert pickle.loads(pickles[backend]) == out
        if backend == "device":   # read back by the host path
            assert tc.corrupt(list(corpus), 0.5, 1, backend="host") == out
    assert pickles["host"] == pickles["device"]


def _outcome(fn):
    try:
        return "ok", fn()
    except Exception as e:           # noqa: BLE001 — the exception itself is what is compared
        return "raised", (type(e), str(e))


@pytest.mark.parametrize("corpus_texts", [["tiny cat and dog"], ["lonely and the cat"], ["lonely lonely spaces"],
                                          ["apple apply ample amply maple mapped"],
                                          ["apple apply ample amply maple mapped couple"]])
def test_tiny_dictionaries_give_the_host_strings_or_its_exception(tmp_path, corpus_texts):
    th = _thesaurus(tmp_path)
    tc = T.TextCorruptor(corpus_texts, cache_dir=None, dictionary_size=6, thesaurus_path=th)
    assert len(tc.common_words) in (0, 1, 2, 6)
    texts = corpus_texts + ["x " + " ".join(tc.common_words * 3), "", "Lonely LONELY lonely"]
    for sev in (0.5, 1.0):
        for w in (None, T.CorruptionWeights(0, 0, 1, 0), T.CorruptionWeights(0, 1, 0, 0)):
            for seed in (0, 5):
                host = _outcome(lambda: tc.corrupt(texts, sev, seed, weights=w, backend="host"))
                dev = _outcome(lambda: tc.corrupt(texts, sev, seed, weights=w, backend="device"))
                assert dev == host, (len(tc.common_words), sev, w, seed)


def test_refused_inputs_raise_before_any_launch(tc):
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="seed"):
        tc.corrupt(["a text"], 0.5, -1, backend="device")
    with pytest.raises(ValueError, match="seed"):
        tc.corrupt(["a text"], 0.5, 2 ** 63 - 10 ** 6, backend="device")
    with pytest.raises(TypeError):
        tc.corrupt(["a text"], 0.5, None, backend="device")
    assert _lib.launch_count() == before
    bad = ["fine text", "lone \ud800 surrogate"]
    host = _outcome(lambda: tc.corrupt(bad, 0.5, 0, backend="host"))
    assert host[0] == "raised" and host[1][0] is UnicodeEncodeError
    assert _outcome(lambda: tc.corrupt(bad, 0.5, 0, backend="device")) == host
    w = T.CorruptionWeights(-1.0, 1.0, 1.0, 1.0)
    assert _outcome(lambda: tc.corrupt(["", "two words"], 0.5, 0, weights=w, backend="device")) == \
        _outcome(lambda: tc.corrupt(["", "two words"], 0.5, 0, weights=w, backend="host"))
