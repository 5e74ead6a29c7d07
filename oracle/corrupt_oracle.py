"""IMDB-C's corruption draws restated in pure Python (TEST INFRASTRUCTURE ONLY): NumPy's SeedSequence -> PCG64
(default_rng), its random(), buffered uint32 draws, the masked-rejection interval behind Generator.shuffle,
Generator.choice(a, p=...), and the md5-mod hashes of text_corruptor.py.  `corrupt` rebuilds
TextCorruptor.corrupt from these draws alone and the corruptor's tables, so that the tests can show that this
restatement (the one the device kernels implement, include/b200tip.h tip_corrupt_*) is complete.
"""
from __future__ import annotations

import hashlib
import re
import string
from typing import List, Sequence

M32, M64, M128 = (1 << 32) - 1, (1 << 64) - 1, (1 << 128) - 1
PCG_MULT = (0x2360ED051FC65DA4 << 64) | 0x4385DF649FCCF645

# SeedSequence's hash constants (numpy/random/bit_generator.pyx)
INIT_A, MULT_A, INIT_B, MULT_B = 0x43B0D7E5, 0x931E8875, 0x8B51F9DD, 0x58F38DED
MIX_MULT_L, MIX_MULT_R, XSHIFT = 0xCA01F9DD, 0x4973F715, 16
POOL_SIZE = 4


def entropy_words(seed: int) -> List[int]:
    """A non-negative int as SeedSequence reads it: little-endian uint32 words, [0] for 0."""
    if seed < 0:
        raise ValueError("expected non-negative integer")
    words = [] if seed else [0]
    while seed:
        words.append(seed & M32)
        seed >>= 32
    return words


def seed_sequence_state(seed: int, n_words64: int = 4) -> List[int]:
    """SeedSequence(seed).generate_state(n_words64, np.uint64)."""
    ent = entropy_words(seed)
    hc = INIT_A

    def hashmix(v):
        nonlocal hc
        v = (v ^ hc) & M32
        hc = (hc * MULT_A) & M32
        v = (v * hc) & M32
        return v ^ (v >> XSHIFT)

    def mix(x, y):
        r = (MIX_MULT_L * x - MIX_MULT_R * y) & M32
        return r ^ (r >> XSHIFT)

    pool = [hashmix(ent[i] if i < len(ent) else 0) for i in range(POOL_SIZE)]
    for s in range(POOL_SIZE):
        for d in range(POOL_SIZE):
            if s != d:
                pool[d] = mix(pool[d], hashmix(pool[s]))
    for s in range(POOL_SIZE, len(ent)):
        for d in range(POOL_SIZE):
            pool[d] = mix(pool[d], hashmix(ent[s]))
    hb = INIT_B
    out32 = []
    for i in range(2 * n_words64):
        v = (pool[i % POOL_SIZE] ^ hb) & M32
        hb = (hb * MULT_B) & M32
        v = (v * hb) & M32
        out32.append(v ^ (v >> XSHIFT))
    return [out32[2 * i] | (out32[2 * i + 1] << 32) for i in range(n_words64)]


class PCG64:
    """default_rng(seed)'s bit generator: PCG64 (XSL-RR 128/64) seeded through SeedSequence."""

    def __init__(self, seed: int):
        w = seed_sequence_state(seed)
        initstate, initseq = (w[0] << 64) | w[1], (w[2] << 64) | w[3]
        self.inc = ((initseq << 1) | 1) & M128
        self.state = 0
        self._step()
        self.state = (self.state + initstate) & M128
        self._step()
        self.has_u32, self.u32 = False, 0

    def _step(self):
        self.state = (self.state * PCG_MULT + self.inc) & M128

    def next64(self) -> int:
        self._step()
        x = ((self.state >> 64) ^ self.state) & M64
        rot = self.state >> 122
        return ((x >> rot) | (x << ((64 - rot) & 63))) & M64

    def next32(self) -> int:
        """Buffered: one next64 gives its low half, then its high half."""
        if self.has_u32:
            self.has_u32 = False
            return self.u32
        v = self.next64()
        self.has_u32, self.u32 = True, v >> 32
        return v & M32

    def random(self) -> float:
        return (self.next64() >> 11) * (1.0 / 9007199254740992.0)

    def interval(self, mx: int) -> int:
        """random_interval(max): masked rejection, on uint32 draws while max fits in 32 bits."""
        if mx == 0:
            return 0
        mask = (1 << mx.bit_length()) - 1
        draw = self.next32 if mx <= M32 else self.next64
        while True:
            v = draw() & mask
            if v <= mx:
                return v

    def shuffle(self, x: list) -> None:
        for i in range(len(x) - 1, 0, -1):
            j = self.interval(i)
            x[i], x[j] = x[j], x[i]


def choice_cdf(p: Sequence[float]):
    """Generator.choice's cdf of p: p.cumsum() / its last entry, in float64 (NumPy's cumsum is sequential)."""
    import numpy as np

    cdf = np.asarray(p, dtype=np.float64).cumsum()
    cdf /= cdf[-1]
    return [float(c) for c in cdf]


def search_right(cdf: Sequence[float], u: float) -> int:
    """cdf.searchsorted(u, side="right") of a sorted cdf: the entries <= u (NaN entries never are)."""
    return sum(1 for c in cdf if c <= u)


def choice(rng: PCG64, a: Sequence, p: Sequence[float]):
    if len(a) == 0:
        raise ValueError("a cannot be empty unless no samples are taken")
    return a[search_right(choice_cdf(p), rng.random())]


def md5_mod(msg: bytes) -> int:
    return int(hashlib.md5(msg).hexdigest(), 16) % 1000000


def split(text: str) -> List[str]:
    return re.findall(r"\w+|[^\w\s]+", text)


# ---- TextCorruptor.corrupt on these draws ----------------------------------------------------------------------
def _typo(w: str, seed: int) -> str:
    k = seed % len(w)
    letters = string.ascii_lowercase.replace(w[k], "")
    return w[:k] + letters[md5_mod(f"{w} {seed}".encode()) % len(letters)] + w[k + 1:]


def _autocorrect(tc, w: str, seed: int) -> str:
    k = tc._word_index.get(w)
    if k is None:
        return w
    import numpy as np

    idx = np.argsort(tc.lev_dist[k])[1:6]
    d = 1 / tc.lev_dist[k][idx]
    return tc.common_words[int(choice(PCG64(seed), [int(i) for i in idx], d / d.sum()))]


def _autocomplete(tc, w: str, seed: int) -> str:
    for n in range(min(5, len(w)), 2, -1):
        bag = [b for b in tc.start_bags.get(n, {}).get(w[:n], []) if b != w]
        if bag:
            return bag[md5_mod(f"{w} {seed}".encode()) % len(bag)]
    return _autocorrect(tc, w, seed)


def _synonym(tc, w: str, seed: int) -> str:
    syn = tc.thesaurus.get(w)
    if not syn:
        return _typo(w, seed)
    return syn[md5_mod(f"{w} {seed} _corrupt_synonym".encode()) % len(syn)]


def corrupt(tc, texts: Sequence[str], severity: float, seed: int, weights=None) -> List[str]:
    """TextCorruptor.corrupt (no cache) of the corruptor `tc`'s tables, every draw from this module."""
    import numpy as np

    w = (0.05, 0.30, 0.30, 0.35) if weights is None else (weights.typo_weight, weights.autocomplete_weight,
                                                          weights.autocorrect_weight, weights.synonym_weight)
    w = np.array(w)
    type_cdf = choice_cdf(w / w.sum())
    out = []
    for text in texts:
        words = split(text)
        n = len(words)
        s = md5_mod(" ".join(words).encode()) + seed
        rng = PCG64(s)
        types = [search_right(type_cdf, rng.random()) for _ in range(n)]
        order = list(range(n))
        PCG64(s).shuffle(order)
        chosen = set(order[: round(n * severity)])
        new = []
        for i, word in enumerate(words):
            if i not in chosen or len(word) < 2:
                new.append(word)
                continue
            # the type index k is CorruptionType(k): TYPO, SYNONYM, AUTOCOMPLETE, AUTOCORRECT
            fn = (lambda a, b, c: _typo(b, c), _synonym, _autocomplete, _autocorrect)[types[i]]
            new.append(fn(tc, word, s + i))
        out.append(" ".join(new))
    return out
