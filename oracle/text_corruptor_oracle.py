"""IMDB-C's TextCorruptor: independent distances, the unmodified reference, a synthetic corpus and its golden file
(TEST INFRASTRUCTURE ONLY).

* `levenshtein_matrix` — the plain DP of oracle/lev_oracle.c over raw code points (built by `build()`, which
  __graft_entry__.build() calls), fast enough to check a full 4 000-word matrix.
* `polyleven_levenshtein` — a pure-Python DP restatement of polyleven.levenshtein(a, b), the C extension the
  reference imports (not installable offline).  With it, `reference()` imports the reference's
  src/core/text_corruptor.py unmodified; `tqdm` and `datasets` import as they are, the module's `load_dataset`
  is replaced by a function that raises, and while the context is open `urllib.request.urlretrieve` raises too,
  so the reference can never reach the network (its load_bad_translations downloads when its cache file is
  missing).
* `synthetic_corpus` — seeded texts drawn Zipf-like from thesaurus headwords, with capitals, digits, punctuation
  runs, `_`, accented and non-BMP characters, words of <= 2 characters and words longer than 64 code points.
* `make_golden()` (python -m oracle.text_corruptor_oracle) — runs the reference on that corpus under
  PYTHONHASHSEED=0 and writes tests/golden/text_corruptor_reference.npz and the thesaurus subset
  tests/golden/text_corruptor_thesaurus.jsonl.  Needs the reference tree (ref_harness.REFERENCE_ROOT).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import types
import urllib.request

import numpy as np

from oracle import ref_harness

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lev_oracle.c")
_SO = os.path.join(_HERE, "liblevoracle.so")
ROOT = os.path.dirname(_HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden", "text_corruptor_reference.npz")
THESAURUS_FIXTURE = os.path.join(ROOT, "tests", "golden", "text_corruptor_thesaurus.jsonl")
GOLDEN_SEVERITIES = (0.0, 0.1, 0.5, 1.0)
GOLDEN_SEEDS = (0, 1)
GOLDEN_WEIGHTS = dict(typo_weight=0.4, autocomplete_weight=0.1, autocorrect_weight=0.2, synonym_weight=0.3)
# dictionary sizes of the two golden configurations: below and above the corpus's distinct eligible words
GOLDEN_SIZES = {"small": 250, "large": 4000}
_lib = None


# ---- the C DP --------------------------------------------------------------------------------------------------
def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.run(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", _SRC, "-o", _SO], check=True)
    return _SO


def _load():
    global _lib
    if _lib is None:
        build()
        lib = C.CDLL(_SO)
        vp, i64 = C.c_void_p, C.c_int64
        lib.oracle_levenshtein.argtypes = [vp, vp, i64, vp, vp, i64, vp, C.c_int]
        lib.oracle_levenshtein.restype = None
        lib.oracle_lev_max_threads.restype = C.c_int
        _lib = lib
    return _lib


def _code_points(words):
    lengths = np.fromiter(map(len, words), dtype=np.int64, count=len(words))
    off = np.zeros(len(words) + 1, dtype=np.int64)
    np.cumsum(lengths, out=off[1:])
    cps = np.frombuffer("".join(words).encode("utf-32-le", "surrogatepass"), dtype="<u4").astype(np.int32)
    return np.concatenate([cps, np.zeros(1, np.int32)]), off


def levenshtein_matrix(a_words, b_words=None) -> np.ndarray:
    """int32 [len(a), len(b)] Levenshtein distances by the plain DP (b None: a against itself)."""
    b_words = a_words if b_words is None else b_words
    a_ids, a_off = _code_points(list(a_words))
    b_ids, b_off = _code_points(list(b_words))
    out = np.zeros((len(a_off) - 1, len(b_off) - 1), dtype=np.int32)
    if out.size:
        lib = _load()
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        lib.oracle_levenshtein(p(a_ids), p(a_off), out.shape[0], p(b_ids), p(b_off), out.shape[1], p(out),
                               lib.oracle_lev_max_threads())
    return out


# ---- the reference ---------------------------------------------------------------------------------------------
def polyleven_levenshtein(a: str, b: str, k=None) -> int:
    """polyleven.levenshtein(a, b): unit-cost edit distance of two str, by code point (the bound k is not used
    by the reference)."""
    row = list(range(len(b) + 1))
    for x, ca in enumerate(a, 1):
        diag, row[0] = row[0], x
        for y, cb in enumerate(b, 1):
            up = row[y]
            row[y] = min(diag + (ca != cb), up + 1, row[y - 1] + 1)
            diag = up
    return row[len(b)]


def _polyleven_stub() -> types.ModuleType:
    m = types.ModuleType("polyleven")
    m.levenshtein = polyleven_levenshtein
    return m


def _refuse_network(*args, **kwargs):
    raise RuntimeError("the reference text_corruptor tried to download; tests never reach the network")


_ref_module = None


@contextlib.contextmanager
def reference():
    """The reference's src/core/text_corruptor.py module (unmodified, on the polyleven stub); inside the context
    urllib.request.urlretrieve raises."""
    global _ref_module
    if not ref_harness.available():
        raise RuntimeError(f"reference not found under {ref_harness.REFERENCE_ROOT}")
    if _ref_module is None:
        sys.modules.setdefault("polyleven", _polyleven_stub())
        path = os.path.join(ref_harness.REFERENCE_ROOT, "src", "core", "text_corruptor.py")
        spec = importlib.util.spec_from_file_location("tip_ref_text_corruptor", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.load_dataset = _refuse_network
        _ref_module = mod
    saved = urllib.request.urlretrieve
    urllib.request.urlretrieve = _refuse_network
    try:
        yield _ref_module
    finally:
        urllib.request.urlretrieve = saved


def seed_reference_cache(cache_dir: str, base_dataset, dictionary_size: int, thesaurus_jsonl: str) -> str:
    """Places the thesaurus where the reference's TextCorruptor looks for its cache file
    (<cache_dir>/<md5 of base_dataset + [str(size)]>/bad_translations.pkl), so that it never downloads."""
    import hashlib
    import shutil

    digest = hashlib.md5(" ".join(list(base_dataset) + [str(dictionary_size)]).encode("utf-8")).hexdigest()
    d = os.path.join(cache_dir, digest)
    os.makedirs(d, exist_ok=True)
    shutil.copyfile(thesaurus_jsonl, os.path.join(d, "bad_translations.pkl"))
    return d


# ---- the synthetic corpus --------------------------------------------------------------------------------------
_ODD_WORDS = ["café", "naïve", "résumé", "über", "façade", "crème", "fiancée", "𝔘nicode", "𝒮cript", "smile𝟘𝟙",
              "snake_case", "__init__", "x_y_z", "2nd", "1999", "42", "3d", "mp3s", "HELLO", "Movie"]
_PUNCT = ["...", "!?", "--", ",", ".", "!!!", "(", ")", "'", "\"", ":-)", "😀😀", "…"]
_SHORT = ["a", "an", "of", "it", "is", "to", "I", "ok", "we", "go"]
_LONG = ["antidisestablishmentarian" * 3, "pneumonoultramicroscopic" * 5 + "silicovolcanoconiosis",
         "x" + "abcdefghij" * 6 + "xyz"]   # 75, 141 and 64 code points: the kernel's blocked path and its edge


def thesaurus_headwords(path: str, count: int, seed: int):
    """`count` seeded single-token alphabetic headwords of a thesaurus .jsonl (each line's "word")."""
    words = []
    with open(path) as f:
        for line in f:
            w = json.loads(line)["word"]
            if w.isalpha() and w.isascii() and 3 <= len(w) <= 14:
                words.append(w)
    words = sorted(set(words))
    rng = np.random.default_rng(seed)
    return [words[k] for k in np.sort(rng.choice(len(words), size=count, replace=False))]


def synthetic_corpus(vocab, n_texts: int, seed: int, mean_len: int = 40):
    """Seeded texts: words drawn Zipf-like from vocab (so that counts tie and most_common has to break ties),
    some capitalised, mixed with the odd words, short words, punctuation runs and a few long words."""
    rng = np.random.default_rng(seed)
    vocab = list(vocab)
    zipf = 1.0 / np.arange(1, len(vocab) + 1) ** 1.05
    zipf /= zipf.sum()
    texts = []
    for _ in range(n_texts):
        n = int(rng.integers(mean_len // 4, mean_len * 2))
        toks = []
        for _ in range(n):
            u = rng.random()
            if u < 0.72:
                w = vocab[int(rng.choice(len(vocab), p=zipf))]
                if rng.random() < 0.1:
                    w = w.capitalize()
            elif u < 0.82:
                w = _SHORT[int(rng.integers(len(_SHORT)))]
            elif u < 0.90:
                w = _PUNCT[int(rng.integers(len(_PUNCT)))]
            elif u < 0.985:
                w = _ODD_WORDS[int(rng.integers(len(_ODD_WORDS)))]
            else:
                w = _LONG[int(rng.integers(len(_LONG)))]
            toks.append(w)
        texts.append(" ".join(toks))
    return texts


def thesaurus_subset(path: str, corpus, out_path: str) -> int:
    """Writes the lines of the thesaurus whose "word" is a token of the corpus (as split_by_whitespace splits)."""
    import re

    tokens = {t for text in corpus for t in re.findall(r"\w+|[^\w\s]+", text)}
    n = 0
    with open(path) as f, open(out_path, "w") as g:
        for line in f:
            if json.loads(line)["word"] in tokens:
                g.write(line)
                n += 1
    return n


def golden_corpus():
    return synthetic_corpus(thesaurus_headwords(
        os.path.join(ref_harness.REFERENCE_ROOT, "datasets", "en_thesaurus.jsonl"), 400, seed=11), 200, seed=12,
        mean_len=30)


# ---- the golden file -------------------------------------------------------------------------------------------
def _json(obj) -> np.ndarray:
    """A 0-d unicode array holding obj as JSON (loads with allow_pickle=False; dict order is kept)."""
    return np.array(json.dumps(obj, ensure_ascii=False))


def golden_value(golden, key):
    return json.loads(str(golden[key]))


def make_golden() -> str:
    """Runs the reference's TextCorruptor on the golden corpus under PYTHONHASHSEED=0 (re-executing itself in a
    subprocess when the hash seed differs: the synonym lists are list(set(...)) of str)."""
    if os.environ.get("PYTHONHASHSEED") != "0":
        env = dict(os.environ, PYTHONHASHSEED="0")
        subprocess.run([sys.executable, "-m", "oracle.text_corruptor_oracle"], check=True, cwd=ROOT, env=env)
        return GOLDEN
    corpus = golden_corpus()
    thesaurus_subset(os.path.join(ref_harness.REFERENCE_ROOT, "datasets", "en_thesaurus.jsonl"), corpus,
                     THESAURUS_FIXTURE)
    out = {"corpus": _json(corpus)}
    with reference() as ref, tempfile.TemporaryDirectory() as tmp:
        for name, size in GOLDEN_SIZES.items():
            seed_reference_cache(tmp, corpus, size, THESAURUS_FIXTURE)
            tc = ref.TextCorruptor(corpus, cache_dir=tmp, dictionary_size=size)
            out[f"{name}_common_words"] = _json(tc.common_words)
            out[f"{name}_start_bags"] = _json(tc.start_bags)
            out[f"{name}_distances"] = tc.lev_dist
            for sev in GOLDEN_SEVERITIES:
                for seed in GOLDEN_SEEDS:
                    out[f"{name}_corrupt_{sev}_{seed}"] = _json(tc.corrupt(corpus, sev, seed))
            out[f"{name}_corrupt_weights"] = _json(
                tc.corrupt(corpus, 0.5, 0, weights=ref.CorruptionWeights(**GOLDEN_WEIGHTS), force_recalculate=True))
    np.savez_compressed(GOLDEN, **out)
    return GOLDEN


if __name__ == "__main__":
    print(make_golden())
