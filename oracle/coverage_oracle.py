"""Exact references for the coverage kernels of csrc/coverage.cu (TEST INFRASTRUCTURE ONLY; NumPy only).

  * `pack_cover` / `unpack_cover`: the packed profile layout of tip_cover_threshold / tip_tknc — neurons in groups
    of 128, word 4*g + i of a row holds in bit l the entry of neuron 128*g + 4*l + i; NBC has two planes (lower
    boundary first).  `pack_plain`: tip_pack_bool's layout, bit b of word w = entry 32*w + b.
  * `tknc_exact`: neuron_coverage.py:159-173 with a STABLE ascending argsort, i.e. the kernel's documented rule for
    equal values (the higher index is marked; NaN sorts above everything), for any integer k (the slice `[-k:]`
    is Python's, so k = 0 marks every neuron and k < 0 all but the |k| lowest).
  * `welford_from`: welford==0.2.5's `add` (count += 1; delta = x - m; m += delta / count; s += delta * (x - m))
    sample by sample from an arbitrary state, in the activation dtype; NumPy turns the Python-int count into the
    array's dtype before dividing, so the restatement divides by `dtype(count)`.
  * `cam_greedy`: the greedy part of prioritizers.py:16-45 (np_oracle.cam_oracle), the picks only.

The private helpers `_grid`, `_top_order`, `_count_as` and `_first_argmax` hold the one rule each function is about,
so that tests/test_coverage_oracle.py can swap in a defective rule and check that the comparisons notice.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def _score_dtype(total: int):
    return np.int16 if total <= np.iinfo(np.int16).max else (np.int32 if total <= np.iinfo(np.int32).max else np.int64)


# ---- packed layouts ----------------------------------------------------------------------------------------------
def packed_words(d: int) -> int:
    """tip_cover_packed_words: words per row and plane"""
    return 4 * (-(-d // 128))


def _grid(a: np.ndarray) -> np.ndarray:
    """[n, 128*G] neuron-major -> [n, G, 32 (bit l), 4 (word i)] view: neuron 128*g + 4*l + i"""
    n, w = a.shape
    return a.reshape(n, w // 128, 32, 4)


def pack_cover(profile) -> np.ndarray:
    """Dense profile [n, d] (NAC / SNAC / TKNC) or [n, d, 2] (NBC) -> uint32 [n, planes * packed_words(d)]"""
    p = np.asarray(profile).astype(bool)
    if p.ndim == 3:
        return np.concatenate([pack_cover(p[..., 0]), pack_cover(p[..., 1])], axis=1)
    n, d = p.shape
    words = packed_words(d)
    pad = np.zeros((n, 32 * words), dtype=np.uint32)
    pad[:, :d] = p
    shifted = _grid(pad) << np.arange(32, dtype=np.uint32)[None, None, :, None]
    return np.bitwise_or.reduce(shifted, axis=2).reshape(n, words)


def unpack_cover(bits, d: int, planes: int = 1) -> np.ndarray:
    """Inverse of pack_cover: [n, planes * packed_words(d)] -> bool [n, d] (planes = 1) or [n, d, 2] (planes = 2).
    Padding bits are dropped; `pack_cover(unpack_cover(b, d)) == b` holds exactly when they are all 0."""
    b = np.asarray(bits).view(np.uint32) if np.asarray(bits).dtype != np.uint32 else np.asarray(bits)
    n = b.shape[0]
    words = packed_words(d)
    assert b.shape[1] == planes * words, (b.shape, d, planes)
    out = []
    for p in range(planes):
        w = b[:, p * words:(p + 1) * words].reshape(n, words // 4, 1, 4)
        flat = np.empty((n, 32 * words), dtype=bool)
        _grid(flat)[...] = (w >> np.arange(32, dtype=np.uint32)[None, None, :, None]) & 1
        out.append(flat[:, :d])
    return out[0] if planes == 1 else np.stack(out, axis=2)


def pack_plain(profile) -> np.ndarray:
    """tip_pack_bool: entries [n, f] (non-zero = covered) -> uint32 [n, ceil(f / 32)], bit b of word w = entry 32w+b"""
    p = np.asarray(profile).reshape(np.asarray(profile).shape[0], -1) != 0
    n, f = p.shape
    words = -(-f // 32)
    pad = np.zeros((n, 32 * words), dtype=bool)
    pad[:, :f] = p
    # bit b of byte j = entry 8j + b; four bytes read as one little-endian word = entries 32w .. 32w + 31
    return np.ascontiguousarray(np.packbits(pad, axis=1, bitorder="little")).view("<u4").astype(np.uint32)


# ---- TKNC --------------------------------------------------------------------------------------------------------
def _top_order(flat: np.ndarray) -> np.ndarray:
    """ascending order per row; equal values keep index order (so the higher index ranks higher), NaN last"""
    return np.argsort(flat, axis=1, kind="stable")


def tknc_count(k: int, d: int) -> int:
    """neurons the reference marks in a layer of d: len(range(d)[-k:])"""
    return len(range(d)[-int(k):])


def tknc_exact(k: int, layers: Sequence[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
    """(scores, profile) of TKNC(k) with the kernel's tie rule; scores in sum_score's dtype"""
    per_layer = []
    for layer in layers:
        flat = np.asarray(layer).reshape(np.asarray(layer).shape[0], -1)
        top = _top_order(flat)[..., -int(k):]
        mark = np.zeros(flat.shape, dtype=bool)
        np.put_along_axis(mark, top, True, axis=1)
        per_layer.append(mark)
    prof = np.concatenate(per_layer, axis=1)
    return np.sum(prof, axis=1, dtype=_score_dtype(prof.shape[1])), prof


# ---- Welford -----------------------------------------------------------------------------------------------------
def _count_as(t, count: int):
    """the count as NumPy divides by it: converted to the state's dtype"""
    return t(count)


def welford_from(x, count_before: int, mean, m2, mn, mx):
    """tip_stats_update's result: x [n, d] folded into the state (count_before samples so far; mean, m2, mn, mx of
    x's dtype) one sample at a time.  Returns new copies (mean, m2, mn, mx)."""
    x = np.asarray(x)
    t = x.dtype.type
    m, s = np.array(mean, dtype=t), np.array(m2, dtype=t)
    lo, hi = np.array(mn, dtype=t), np.array(mx, dtype=t)
    count = int(count_before)
    with np.errstate(all="ignore"):
        for r in range(x.shape[0]):
            count += 1
            c = _count_as(t, count)
            # one IEEE operation per ufunc, element by element over the neurons (NumPy contracts nothing into FMAs)
            delta = (x[r] - m).astype(t)
            m = (m + (delta / c).astype(t)).astype(t)
            s = (s + (delta * (x[r] - m).astype(t)).astype(t)).astype(t)
            lo = np.minimum(lo, x[r])
            hi = np.maximum(hi, x[r])
    return m, s, lo, hi


# ---- CAM ---------------------------------------------------------------------------------------------------------
def _first_argmax(gain: np.ndarray) -> int:
    return int(np.argmax(gain))


def cam_greedy(profile) -> np.ndarray:
    """The greedy picks of cam (prioritizers.py:24-45): pick the sample with the most still-uncovered entries (first
    index on ties) until the best gain is 0.  profile: bool [n, ...]."""
    prof = np.asarray(profile).reshape(np.asarray(profile).shape[0], -1).astype(bool)
    covered = np.zeros(prof.shape[1], dtype=bool)
    gain = prof.sum(axis=1).astype(np.int64)
    order: List[int] = []
    while prof.shape[0] and len(order) < prof.shape[0]:
        pick = _first_argmax(gain)
        if gain[pick] <= 0:
            break
        order.append(pick)
        fresh = prof[pick] & ~covered
        covered |= fresh
        gain = gain - prof[:, fresh].sum(axis=1)
    return np.asarray(order, dtype=np.int64)
