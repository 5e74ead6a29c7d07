"""CPU tests of the IMDB-C generator (simple_tip_b200.core.text_corruptor): with the dictionary's distances cached
the whole class runs on the host, so it is checked here against the reference's golden outputs, against the
unmodified reference in one process (skipped without it) and for cache compatibility in both directions."""
import json
import os
import subprocess
import sys
import urllib.request

import numpy as np
import pytest

from oracle import ref_harness
from oracle import text_corruptor_oracle as TO
from simple_tip_b200 import _lib
from simple_tip_b200.core import text_corruptor as T

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
needs_reference = pytest.mark.skipif(not ref_harness.available(), reason="reference tree not present")

# Runs in a PYTHONHASHSEED=0 interpreter (the synonym lists follow the hash seed): builds the port on the golden
# corpus for both dictionary sizes, with distances.npy pre-placed from the golden (argv[1] == "cached") or computed
# on the device, and prints {key: equal to the golden}.
GOLDEN_CHECK = r"""
import json, os, sys, tempfile
import numpy as np
sys.path.insert(0, os.getcwd())
from oracle import text_corruptor_oracle as TO
from src.core.text_corruptor import CorruptionWeights, TextCorruptor
g = np.load(TO.GOLDEN, allow_pickle=False)
corpus = TO.golden_value(g, "corpus")
res = {}
with tempfile.TemporaryDirectory() as tmp:
    for name, size in TO.GOLDEN_SIZES.items():
        if sys.argv[1] == "cached":
            d = TO.seed_reference_cache(tmp, corpus, size, TO.THESAURUS_FIXTURE)
            os.remove(os.path.join(d, "bad_translations.pkl"))
            np.save(os.path.join(d, "distances.npy"), g[f"{name}_distances"])
        tc = TextCorruptor(corpus, cache_dir=tmp, dictionary_size=size, thesaurus_path=TO.THESAURUS_FIXTURE)
        res[f"{name}_distances"] = bool(np.array_equal(tc.lev_dist, g[f"{name}_distances"])
                                        and tc.lev_dist.dtype == np.uint8)
        res[f"{name}_common_words"] = tc.common_words == TO.golden_value(g, f"{name}_common_words")
        for sev in TO.GOLDEN_SEVERITIES:
            for seed in TO.GOLDEN_SEEDS:
                key = f"{name}_corrupt_{sev}_{seed}"
                res[key] = tc.corrupt(corpus, sev, seed) == TO.golden_value(g, key)
        got = tc.corrupt(corpus, 0.5, 0, weights=CorruptionWeights(**TO.GOLDEN_WEIGHTS), force_recalculate=True)
        res[f"{name}_corrupt_weights"] = got == TO.golden_value(g, f"{name}_corrupt_weights")
print(json.dumps(res))
"""


def run_golden_check(mode: str) -> dict:
    env = dict(os.environ, PYTHONHASHSEED="0")
    out = subprocess.run([sys.executable, "-c", GOLDEN_CHECK, mode], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def gold():
    return np.load(TO.GOLDEN, allow_pickle=False)


def _cached_port(tmp, corpus, size, distances, **kw):
    """A port TextCorruptor whose distances.npy is pre-placed (so it needs no device)."""
    d = os.path.join(tmp, T._hash_text_to_str(list(corpus) + [str(size)]))
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, "distances.npy"), np.asarray(distances, dtype=np.uint8))
    return T.TextCorruptor(list(corpus), cache_dir=tmp, dictionary_size=size, **kw)


def test_port_reproduces_the_golden_corruptions_under_hash_seed_0():
    res = run_golden_check("cached")
    assert res and all(res.values()), [k for k, v in res.items() if not v]


@pytest.mark.parametrize("name", sorted(TO.GOLDEN_SIZES))
def test_common_words_and_start_bags_match_the_golden(gold, tmp_path, name):
    corpus = TO.golden_value(gold, "corpus")
    tc = _cached_port(str(tmp_path), corpus, TO.GOLDEN_SIZES[name], gold[f"{name}_distances"],
                      thesaurus_path=TO.THESAURUS_FIXTURE)
    assert tc.common_words == TO.golden_value(gold, f"{name}_common_words")
    assert json.dumps(tc.start_bags, ensure_ascii=False) == str(gold[f"{name}_start_bags"])   # order included
    if name == "large":   # dictionary_size above the distinct eligible words: every one of them is kept
        assert len(tc.common_words) < TO.GOLDEN_SIZES[name]


@pytest.mark.parametrize("weights", [T.CorruptionWeights(), T.CorruptionWeights(0.4, 0.1, 0.2, 0.3),
                                     T.CorruptionWeights(1.0, 0.0, 0.0, 0.0), T.CorruptionWeights(1, 2, 3, 4)])
def test_vectorised_type_draws_equal_the_choice_loop(weights):
    w = np.array([weights.typo_weight, weights.autocomplete_weight, weights.autocorrect_weight,
                  weights.synonym_weight])
    p = w / w.sum()
    for seed in (1, 7, 123456, 999999):
        for n in (0, 1, 5, 230, 1000):
            rng = np.random.default_rng(seed)
            want = [T.CorruptionType(rng.choice(4, p=p)) for _ in range(n)]      # text_corruptor.py:144-146
            assert T._generate_corruption_types(seed, n, weights) == want, (seed, n)


def test_missing_thesaurus_raises_and_never_downloads(gold, tmp_path, monkeypatch):
    def no_download(*a, **k):
        pytest.fail("urlretrieve was called")

    monkeypatch.setattr(urllib.request, "urlretrieve", no_download)
    corpus = TO.golden_value(gold, "corpus")
    with pytest.raises(FileNotFoundError, match="THESAURUS_DOWNLOAD"):
        _cached_port(str(tmp_path), corpus, 250, gold["small_distances"])
    with pytest.raises(FileNotFoundError, match="THESAURUS_DOWNLOAD"):
        _cached_port(str(tmp_path), corpus, 250, gold["small_distances"], thesaurus_path=str(tmp_path / "none.jsonl"))
    tc = T.TextCorruptor.__new__(T.TextCorruptor)            # cache_dir=None: the file is read in place
    tc.cache_dir, tc.thesaurus_path = None, None
    with pytest.raises(FileNotFoundError, match="cache_dir=None"):
        tc.load_bad_translations()
    tc.thesaurus_path = TO.THESAURUS_FIXTURE
    assert len(tc.load_bad_translations()) > 0
    # with the thesaurus given, the cache directory gets the reference's file
    tc = _cached_port(str(tmp_path), corpus, 250, gold["small_distances"], thesaurus_path=TO.THESAURUS_FIXTURE)
    with open(os.path.join(tc.cache_dir, "bad_translations.pkl"), "rb") as f, open(TO.THESAURUS_FIXTURE, "rb") as g:
        assert f.read() == g.read()


def test_overlong_words_raise_before_the_device():
    with pytest.raises(ValueError, match=r"word 2 has 256 code points"):
        T._levensthein_distance("abc", ["a", "b", "x" * 256])
    with pytest.raises(ValueError, match=r"word 0 has 300 code points"):
        from simple_tip_b200 import engine as E

        E.levenshtein(["\U0001d518" * 300, "b"])


def test_levenshtein_abi_symbol_is_exported():
    assert "tip_levenshtein" in _lib.symbols()
    assert hasattr(_lib.load(), "tip_levenshtein")


def test_c_dp_agrees_with_the_polyleven_restatement():
    rng = np.random.default_rng(5)
    alphabet = list("abcdé") + ["\U0001d518", "_"]
    words = ["", "a"] + ["".join(rng.choice(alphabet, size=int(rng.integers(0, 30)))) for _ in range(40)]
    want = np.array([[TO.polyleven_levenshtein(a, b) for b in words] for a in words])
    assert np.array_equal(TO.levenshtein_matrix(words), want)


def _vocab():
    with open(TO.THESAURUS_FIXTURE) as f:
        return sorted({json.loads(l)["word"] for l in f if json.loads(l)["word"].isalpha()})


@needs_reference
@pytest.mark.parametrize("seed,size", [(21, 150), (22, 4000), (23, 60)])
def test_port_equals_the_reference_in_one_process(tmp_path, seed, size):
    corpus = TO.synthetic_corpus(_vocab(), 80, seed=seed, mean_len=24)
    words = T.TextCorruptor.__new__(T.TextCorruptor)
    words.cache_dir = None
    dist = TO.levenshtein_matrix(words._extract_common_words(corpus, size)).astype(np.uint8)   # the C DP
    d = TO.seed_reference_cache(str(tmp_path / "ref"), corpus, size, TO.THESAURUS_FIXTURE)
    np.save(os.path.join(d, "distances.npy"), dist)
    port = _cached_port(str(tmp_path / "port"), corpus, size, dist, thesaurus_path=TO.THESAURUS_FIXTURE)
    with TO.reference() as R:
        ref = R.TextCorruptor(corpus, cache_dir=str(tmp_path / "ref"), dictionary_size=size)
        assert ref.common_words == port.common_words and ref.start_bags == port.start_bags
        assert ref.thesaurus == port.thesaurus          # same process: same set order
        for sev in (0.0, 0.3, 0.5, 1.0):
            for s in (0, 5):
                assert port.corrupt(corpus, sev, s) == ref.corrupt(corpus, sev, s), (sev, s)
        for w in ((0.05, 0.3, 0.3, 0.35), (0.0, 0.0, 1.0, 0.0), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0)):
            got = port.corrupt(corpus, 0.7, 3, weights=T.CorruptionWeights(*w), force_recalculate=True)
            want = ref.corrupt(corpus, 0.7, 3, weights=R.CorruptionWeights(*w), force_recalculate=True)
            assert got == want, w


@needs_reference
def test_caches_interoperate_both_ways(tmp_path):
    corpus = TO.synthetic_corpus(_vocab(), 40, seed=31, mean_len=20)
    size = 80
    with TO.reference() as R:
        # the reference's cache (its distances from the polyleven restatement) is read by the port
        TO.seed_reference_cache(str(tmp_path / "a"), corpus, size, TO.THESAURUS_FIXTURE)
        ref = R.TextCorruptor(corpus, cache_dir=str(tmp_path / "a"), dictionary_size=size)
        want = ref.corrupt(corpus, 0.5, 2)
        port = T.TextCorruptor(corpus, cache_dir=str(tmp_path / "a"), dictionary_size=size)   # no device needed
        assert np.array_equal(port.lev_dist, ref.lev_dist) and port.common_words == ref.common_words
        assert port.corrupt(corpus, 0.5, 2) == want
        assert port.corrupt(corpus, 0.5, 4, force_recalculate=True) == ref.corrupt(corpus, 0.5, 4, force_recalculate=True)
        # the port's cache is read by the reference, byte for byte the same files
        port = _cached_port(str(tmp_path / "b"), corpus, size, ref.lev_dist, thesaurus_path=TO.THESAURUS_FIXTURE)
        got = port.corrupt(corpus, 0.5, 2)
        for f in ("common-words.pkl", "word-start-bags.pkl", "distances.npy", "bad_translations.pkl",
                  os.path.join("corrupted", os.listdir(os.path.join(port.cache_dir, "corrupted"))[0])):
            with open(os.path.join(port.cache_dir, f), "rb") as x, open(os.path.join(ref.cache_dir, f), "rb") as y:
                assert x.read() == y.read(), f
        ref2 = R.TextCorruptor(corpus, cache_dir=str(tmp_path / "b"), dictionary_size=size)
        assert ref2.common_words == port.common_words and np.array_equal(ref2.lev_dist, port.lev_dist)
        assert ref2.corrupt(corpus, 0.5, 2) == got == want
