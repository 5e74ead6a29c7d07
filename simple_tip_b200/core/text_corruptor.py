"""`src.core.text_corruptor` of the reference (the generator of IMDB-C), with the dictionary's all-pairs Levenshtein
matrix computed on the GPU (tip_levenshtein) and everything else on the host, bit for bit.

Line references are to the reference's src/core/text_corruptor.py.  Where this module differs (DESIGN.md §9):
- the thesaurus is never downloaded: `TextCorruptor(..., thesaurus_path=...)` names a local en_thesaurus.jsonl,
  copied to the reference's cache path when that file is missing; with neither, FileNotFoundError;
- no tqdm progress bars;
- words longer than 255 code points raise ValueError before the distance kernel runs (the reference's uint8 cast of
  such a distance is implementation-defined);
- the corruption loop draws a text's corruption types with one rng.random(n) (what n Generator.choice(4, p=p) calls
  draw), tests membership with a mask, finds word indexes with a dict and memoises each word's autocorrect
  candidates: the same values, without the quadratic steps.
SYNONYM corruptions pick from list(set(...)) of str (:435-444), whose order depends on PYTHONHASHSEED: like the
reference's, they are reproducible only under a fixed hash seed.

corrupt(..., backend="device") (or B200TIP_CORRUPT=device) runs the corruption loop on the GPU (csrc/corrupt.cu):
the same strings, the same cache file.  It refuses seed < 0, and seeds where seed + 10**6 + the longest text's
UTF-8 byte count reaches 2**63, with ValueError before any launch; the host path stays the default.
"""
from __future__ import annotations

import collections
import dataclasses
import enum
import hashlib
import json
import logging
import operator
import os
import pickle
import re
import shutil
import string
import warnings
from typing import Dict, List, Optional

import numpy as np

DEFAULT_CACHE_DIR = "./.text_corruption_cache/"

MAX_COMMON_START_FOR_AUTOCOMPLETE = 5
MIN_COMMON_START_FOR_AUTOCOMPLETE = 3

THESAURUS_DOWNLOAD = (
    "https://raw.githubusercontent.com/zaibacu/thesaurus/master/en_thesaurus.jsonl"
)


def _levensthein_distance(word: str, words: List[str]) -> np.ndarray:
    """:36-51 — float64 [len(words)] Levenshtein distances of `word` to every word of `words` (polyleven's unit
    costs, by code point), one 1 x V row of tip_levenshtein."""
    from .. import engine as E

    return E.levenshtein([word], list(words)).cpu().numpy().reshape(-1).astype(np.float64)


def split_by_whitespace(strings: List[str]) -> List[List[str]]:
    """:54-58 — splits each string with the regex of HuggingFace's WhitespaceSplit."""
    return [re.findall(r"\w+|[^\w\s]+", l) for l in strings]


def bad_autocompletes(
    word: str, start_bags: Dict[int, Dict[str, List[str]]], common_letters: int
) -> Optional[List[str]]:
    """:61-89 — the other words of the start bag of `word`'s first `common_letters` letters, falling back to
    fewer letters (down to MIN_COMMON_START_FOR_AUTOCOMPLETE; below that None)."""
    if common_letters < MIN_COMMON_START_FOR_AUTOCOMPLETE:
        return None
    common_letters = min(common_letters, len(word))
    bag = start_bags.get(common_letters, {}).get(word[:common_letters], [])
    bag = [w for w in bag if w != word]
    if len(bag) == 0:
        return bad_autocompletes(word, start_bags, common_letters=common_letters - 1)
    return bag


class CorruptionType(enum.Enum):
    """:92-107 — the four corruption types."""

    TYPO = 0
    """Randomly replaced single chars. Imitates human typos."""
    SYNONYM = 1
    """Replacement with an (apparent) synonym, ignoring all context (imitates word-by-word translations)."""
    AUTOCOMPLETE = 2
    """Replacement with a word which starts with the same letters as the original word."""
    AUTOCORRECT = 3
    """Replacement with a very similar word (imitates failed mobile phone input pattern recognition)."""


_TYPES = [CorruptionType(k) for k in range(4)]


def _get_rng(seed):
    """:110-115"""
    if seed is None:
        return np.random.default_rng()
    return np.random.default_rng(seed)


@dataclasses.dataclass
class CorruptionWeights:
    """:118-125 — the weights of the corruption types."""

    typo_weight: float = 0.05
    autocomplete_weight: float = 0.30
    autocorrect_weight: float = 0.30
    synonym_weight: float = 0.35


def _generate_corruption_types(
    seed: int,
    num_words: int,
    weights: CorruptionWeights,
) -> List[CorruptionType]:
    """:128-146 — one corruption type per word.  The reference calls rng.choice(4, p=p) num_words times; each call
    draws one double u and returns cdf.searchsorted(u, side="right") with cdf = p.cumsum() / its last entry, so
    one rng.random(num_words) and one searchsorted give the same types from the same generator state."""
    weights = np.array(
        [
            weights.typo_weight,
            weights.autocomplete_weight,
            weights.autocorrect_weight,
            weights.synonym_weight,
        ]
    )
    normalized_weights = weights / weights.sum()
    rng = _get_rng(seed)
    if num_words == 0:
        return []
    if np.any(normalized_weights < 0):          # Generator.choice's own checks
        raise ValueError("probabilities are not non-negative")
    if abs(normalized_weights.sum() - 1.0) > np.sqrt(np.finfo(np.float64).eps):
        raise ValueError("probabilities do not sum to 1")
    cdf = normalized_weights.cumsum()
    cdf /= cdf[-1]
    idx = cdf.searchsorted(rng.random(num_words), side="right")
    return [_TYPES[k] for k in idx]


def _corrupt_backend(backend: Optional[str]) -> str:
    """backend=None: the B200TIP_CORRUPT environment variable, default "host"."""
    backend = backend if backend is not None else os.environ.get("B200TIP_CORRUPT", "host")
    if backend not in ("host", "device"):
        raise ValueError(f"backend must be 'host' or 'device', got {backend!r}")
    return backend


def _hash_text_to_int(words: List[str]) -> int:
    """:149-154"""
    return int(_hash_text_to_str(words), 16) % 1000000


def _hash_text_to_str(words: List[str]) -> str:
    """:157-158"""
    return hashlib.md5(" ".join(words).encode("utf-8")).hexdigest()


class TextCorruptor(object):
    """:161-508 — corrupts arbitrary english text datasets (IMDB-C).  Same constructor and cache layout as the
    reference (caches written by either are read by the other), plus `thesaurus_path`: a local
    en_thesaurus.jsonl used in place of the reference's download."""

    def __init__(
        self,
        base_dataset: List[str],
        cache_dir: Optional[str] = DEFAULT_CACHE_DIR,
        dictionary_size: int = 4000,
        clear_cache: bool = False,
        thesaurus_path: Optional[str] = None,
    ):
        if cache_dir is DEFAULT_CACHE_DIR:
            warnings.warn(
                "Using default cache directory, which is probably not what you want. "
                "Consider passing your own cache dir when creating a "
                "TextCorruptor instance. "
            )
        self.thesaurus_path = thesaurus_path
        self.base_ds_hash: str = _hash_text_to_str(base_dataset + [str(dictionary_size)])
        self.cache_dir: Optional[str] = None
        if cache_dir is not None:
            self.cache_dir = os.path.join(cache_dir, self.base_ds_hash)
            if not os.path.exists(self.cache_dir):
                os.makedirs(self.cache_dir)
            elif clear_cache:
                shutil.rmtree(self.cache_dir)
                os.makedirs(self.cache_dir)

        self.common_words: List[str] = self._extract_common_words(base_dataset, dictionary_size)
        self._word_index = {w: k for k, w in enumerate(self.common_words)}
        self._autocorrect_candidates = {}
        self.start_bags: Dict[int, Dict[str, List[str]]] = self._word_start_bags()
        self.lev_dist: np.ndarray = self._calculate_distances()
        self.thesaurus: Dict[str, List[str]] = self.load_bad_translations()
        self._device_tables = None

    def _cache_file(self, name: str) -> Optional[str]:
        return None if self.cache_dir is None else os.path.join(self.cache_dir, name)

    def _extract_common_words(self, base_dataset: List[str], size: int) -> List[str]:
        """:199-241 — the `size` most common lower-cased words longer than 4 characters that are not numbers and
        contain a letter (Counter.most_common, ties in first-seen order), sorted."""
        words_file = self._cache_file("common-words.pkl")
        if words_file is not None and os.path.exists(words_file):
            logging.info("Loading common words from cache")
            with open(words_file, "rb") as f:
                return pickle.load(f)
        logging.info("Extracting common words")
        words = [w.lower() for l in split_by_whitespace(base_dataset) for w in l]
        words = [w for w in words if len(w) > 4]
        words = [w for w in words if not w.isdigit()]
        words = [w for w in words if any(c.isalpha() for c in w)]
        chosen_words = list(dict(collections.Counter(words).most_common(size)).keys())
        chosen_words.sort()
        logging.info("Finished extracting common words from imdb")
        if words_file is not None:
            with open(words_file, "wb") as f:
                pickle.dump(chosen_words, f)
        return chosen_words

    def _word_start_bags(self) -> Dict[int, Dict[str, List[str]]]:
        """:243-280 — for 3, 4 and 5 start letters, the common words grouped by their start (in word order)."""
        words_bags_file = self._cache_file("word-start-bags.pkl")
        if words_bags_file is not None and os.path.exists(words_bags_file):
            logging.info("Loading word-start-bags from cache")
            with open(words_bags_file, "rb") as f:
                return pickle.load(f)
        result = {}
        for num_start_chars in range(MIN_COMMON_START_FOR_AUTOCOMPLETE, MAX_COMMON_START_FOR_AUTOCOMPLETE + 1):
            bags = dict()
            for word in self.common_words:
                if len(word) >= num_start_chars:
                    bags.setdefault(word[:num_start_chars], []).append(word)
            result[num_start_chars] = bags
        if words_bags_file is not None:
            with open(words_bags_file, "wb") as f:
                pickle.dump(result, f)
        return result

    def _calculate_distances(self) -> np.ndarray:
        """:282-309 — the uint8 [V, V] Levenshtein matrix of the common words, from the cache or from the device
        (tip_levenshtein: each unordered pair once; no CPU fallback).  V = 0 gives shape (0,), as the reference's
        np.array([], dtype=np.uint8)."""
        distances_file = self._cache_file("distances.npy")
        if distances_file is not None and os.path.exists(distances_file):
            logging.info("Loading distances from cache")
            return np.load(distances_file)
        logging.info("Calculating levensthein distances")
        from .. import engine as E

        distances = E.levenshtein(self.common_words).cpu().numpy()
        if len(self.common_words) == 0:
            distances = distances.reshape(0)
        if distances_file is not None:
            np.save(distances_file, distances)
        return distances

    def corrupt(
        self,
        texts: List[str],
        severity: float,
        seed: int,
        weights: Optional[CorruptionWeights] = None,
        force_recalculate: bool = False,
        backend: Optional[str] = None,
    ) -> List[str]:
        """:311-410 — corrupts round(len(words) * severity) words of each text (words shorter than 2 characters
        stay), with per-text seeds from the text's md5, so that a text's corruption depends on neither the other
        texts nor their order, and a higher severity keeps the corruptions of a lower one.  Cached per
        (texts, severity, seed) — not per weights — unless force_recalculate.  backend: "host" (default) or
        "device" (the GPU, string for string the same; None reads B200TIP_CORRUPT)."""
        backend = _corrupt_backend(backend)
        assert 0 <= severity <= 1, "Severity must be between 0 and 1."
        cache_file = None
        if self.cache_dir is not None:
            cache_file = os.path.join(self.cache_dir, "corrupted", f"{_hash_text_to_str(texts)}-{severity}-{seed}.pkl")
            if os.path.exists(cache_file) and not force_recalculate:
                logging.info("Loading corrupted dataset from cache")
                with open(cache_file, "rb") as f:
                    return pickle.load(f)
        if weights is None:
            weights = CorruptionWeights()

        def _corrupt_single_text(words: List[str]) -> str:
            sentence_seed = _hash_text_to_int(words) + seed
            corruption_types = _generate_corruption_types(sentence_seed, len(words), weights)
            corruption_indexes = np.arange(len(words))
            _get_rng(sentence_seed).shuffle(corruption_indexes)
            chosen = np.zeros(len(words), dtype=bool)
            chosen[corruption_indexes[: round(len(words) * severity)]] = True
            new_text = []
            for i, word in enumerate(words):
                if not chosen[i] or len(word) < 2:
                    new_text.append(word)
                else:
                    new_text.append(self._corrupt_word(word, sentence_seed + i, corruption_types[i]))
            return " ".join(new_text)

        if backend == "device":
            corrupted_texts, failed = self._corrupt_on_device(texts, severity, seed, weights)
            if failed is not None:       # the host's exception for the first text that raises there
                _corrupt_single_text(split_by_whitespace([texts[failed]])[0])
                raise RuntimeError(f"the device reported text {failed} as failing, but the host corrupts it")
        else:
            corrupted_texts = [_corrupt_single_text(text) for text in split_by_whitespace(texts)]
        if cache_file is not None:
            os.makedirs(os.path.dirname(cache_file), exist_ok=True)
            with open(cache_file, "wb") as f:
                pickle.dump(corrupted_texts, f)
        return corrupted_texts

    def _corrupt_on_device(self, texts: List[str], severity: float, seed: int, weights: CorruptionWeights):
        """(corrupted texts, None) from the device, or (None, t) when text t is the first for which the host path
        raises (an unencodable text, invalid weights, an autocorrect without candidates)."""
        from .. import engine as E

        seed = operator.index(seed)
        if isinstance(severity, bool) or not isinstance(severity, (int, float)):
            raise TypeError(f"the device backend takes an int or float severity, got {type(severity).__name__}")
        encoded, failed = [], None
        for k, t in enumerate(texts):
            try:
                encoded.append(t.encode("utf-8"))
            except UnicodeEncodeError:
                failed = k
                break
        longest = max(map(len, encoded), default=0)
        if seed < 0 or seed + 10 ** 6 + longest >= 2 ** 63:
            raise ValueError(f"the device backend needs 0 <= seed and seed + 10**6 + {longest} (the longest text's "
                             f"bytes) < 2**63, got seed={seed}")
        w = np.array([weights.typo_weight, weights.autocomplete_weight, weights.autocorrect_weight,
                      weights.synonym_weight])
        normalized_weights = w / w.sum()
        cdf = np.ones(4)                  # used only when no text has words
        if np.any(normalized_weights < 0) or abs(normalized_weights.sum() - 1.0) > np.sqrt(np.finfo(np.float64).eps):
            # _generate_corruption_types raises at the first text with words
            first = next((k for k, t in enumerate(texts[:len(encoded)]) if split_by_whitespace([t])[0]), None)
            if first is not None:
                return None, first
        else:
            cdf = normalized_weights.cumsum()
            cdf /= cdf[-1]
        out, bad = E.corrupt_texts(encoded, self.device_tables(), seed, severity, cdf)
        if bad is not None:
            return None, bad
        if failed is not None:
            return None, failed
        return [b.decode("utf-8", "surrogatepass") for b in out], None

    def _autocorrect_choice(self, word_index: int):
        """(np.argsort(lev_dist[k])[1:6], 1 / distance normalised) of common word k, computed once."""
        cached = self._autocorrect_candidates.get(word_index)
        if cached is None:
            candidate_indices = np.argsort(self.lev_dist[word_index])[1:6]
            candidate_distances = 1 / self.lev_dist[word_index][candidate_indices]
            cached = (candidate_indices, candidate_distances / candidate_distances.sum())
            self._autocorrect_candidates[word_index] = cached
        return cached

    def device_tables(self):
        """The (common words, start bags, thesaurus) tables of the device backend, built on first use and kept."""
        if getattr(self, "_device_tables", None) is None:
            from .. import engine as E

            values, cdfs = [], []
            for k in range(len(self.common_words)):
                candidate_indices, p = self._autocorrect_choice(k)
                values.append([self.common_words[i] for i in candidate_indices])
                if len(p):                # Generator.choice's cdf
                    cdf = p.cumsum()
                    cdf /= cdf[-1]
                    cdfs.append(cdf)
            common = E.CorruptTable(self.common_words, values, np.concatenate(cdfs) if cdfs else np.zeros(0))
            bag_items = [item for n in sorted(self.start_bags) for item in self.start_bags[n].items()]
            bags = E.CorruptTable([key for key, _ in bag_items], [bag for _, bag in bag_items])
            thesaurus = E.CorruptTable(list(self.thesaurus), list(self.thesaurus.values()))
            self._device_tables = (common, bags, thesaurus)
        return self._device_tables

    def load_bad_translations(self) -> Dict[str, List[str]]:
        """:412-446 — {word: list(set(synonyms))} of the thesaurus lines with more than one synonym.  The thesaurus
        is <cache_dir>/bad_translations.pkl (a .jsonl, as the reference names it); when that file is missing,
        `thesaurus_path` is copied there (without a cache dir it is read in place).  Never downloads: with neither
        file, FileNotFoundError."""
        cached = self._cache_file("bad_translations.pkl")
        if cached is not None and os.path.isfile(cached):
            source = cached
        elif self.thesaurus_path is not None and os.path.isfile(self.thesaurus_path):
            source = self.thesaurus_path
            if cached is not None:
                shutil.copyfile(self.thesaurus_path, cached)
                source = cached
        else:
            raise FileNotFoundError(
                f"no thesaurus: {cached or 'no cache file (cache_dir=None)'} is missing and thesaurus_path="
                f"{self.thesaurus_path!r} is not a file.  This port never downloads: fetch THESAURUS_DOWNLOAD "
                f"({THESAURUS_DOWNLOAD}) and pass its path as thesaurus_path.")
        with open(source) as f:
            data = [json.loads(line) for line in f]
        # the reference's literal set / update / list(set) sequence: the list order follows PYTHONHASHSEED
        result = dict()
        for d in data:
            word = d["word"]
            synonyms = d["synonyms"]
            if len(synonyms) > 1:
                if word not in result:
                    result[word] = set()
                result.get(word).update(synonyms)
        for word in result.keys():
            result[word] = list(result.get(word))
        return result

    @staticmethod
    def _corrupt_typo(text, seed: int) -> str:
        """:448-457 — one letter replaced by another lower-case letter, both picked by hash."""
        letter_index = seed % len(text)
        candidate_letters = string.ascii_lowercase.replace(text[letter_index], "")
        random_candidate_index = _hash_text_to_int([text, str(seed)]) % len(candidate_letters)
        typo = candidate_letters[random_candidate_index]
        return text[:letter_index] + typo + text[letter_index + 1:]

    def _corrupt_autocomplete(self, word, seed: int) -> str:
        """:459-466"""
        candidates = bad_autocompletes(word, self.start_bags, common_letters=5)
        if candidates is None or len(candidates) == 0:
            return self._corrupt_autocorrect(word, seed)
        return candidates[_hash_text_to_int([word, str(seed)]) % len(candidates)]

    def _corrupt_autocorrect(self, word, seed: int) -> str:
        """:468-479 — one of the five nearest common words, drawn with probability ~ 1 / distance by a generator
        seeded per word.  The candidates (np.argsort(lev_dist[k])[1:6], NumPy's tie order) and their
        probabilities are computed once per word index."""
        word_index = self._word_index.get(word)
        if word_index is None:
            return word
        candidate_indices, p = self._autocorrect_choice(word_index)
        chosen_index = _get_rng(seed).choice(candidate_indices, p=p)
        return self.common_words[chosen_index]

    def _corrupt_synonym(self, word, seed: int) -> str:
        """:481-496 — a synonym picked by hash, or a typo when the thesaurus has none."""
        synonyms = self.thesaurus.get(word)
        if not synonyms:
            return self._corrupt_typo(word, seed)
        random_candidate_index = _hash_text_to_int([word, str(seed), "_corrupt_synonym"]) % len(synonyms)
        return synonyms[random_candidate_index]

    def _corrupt_word(self, w, seed, corruption_type: CorruptionType) -> str:
        """:498-508"""
        if corruption_type == CorruptionType.TYPO:
            return self._corrupt_typo(w, seed)
        elif corruption_type == CorruptionType.AUTOCOMPLETE:
            return self._corrupt_autocomplete(w, seed)
        elif corruption_type == CorruptionType.AUTOCORRECT:
            return self._corrupt_autocorrect(w, seed)
        elif corruption_type == CorruptionType.SYNONYM:
            return self._corrupt_synonym(w, seed)
        else:
            raise ValueError(f"Unknown corruption type: {corruption_type}")
