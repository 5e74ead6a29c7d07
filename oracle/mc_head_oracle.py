"""NumPy restatement of tip_mc_head (simple_tip_b200/csrc/mc_head.cu) (TEST INFRASTRUCTURE ONLY).

Written from include/b200tip.h's statement of the arithmetic, not from the CUDA:

  * key(l, r, s) = mix(mix(mix(mix(seed) ^ l) ^ r) ^ s) with mix one splitmix64 step (`kmeans_oracle.km_mix`);
    unit j's 32-bit draw is the low (j even) or high (j odd) half of mix(key ^ (j >> 1));
  * unit j is dropped iff u < t, t = rint(p * 2^32); a kept unit is x * scale rounded once to float32, scale =
    float32(1 / float32(1 - p)); a dropped unit is 0;
  * z_c = (((0 + x'_0 K[0, c]) + x'_1 K[1, c]) + ...) + b[c], every product and sum rounded once to float32;
  * relu: z < 0 ? 0 : z; the softmax is restated in float64 (for a bound on the kernel's float32 softmax).

`preact` gives the kernel's TIP_MC_PREACT output bit for bit.  Inputs are NumPy arrays; nothing in the product
package imports this module.
"""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np

F = np.float32
U64 = np.uint64
MASK64 = (1 << 64) - 1


def mix(z: np.ndarray) -> np.ndarray:
    """One splitmix64 step over a uint64 array (wrapping arithmetic)."""
    z = np.asarray(z, dtype=U64)
    with np.errstate(over="ignore"):
        z = z + U64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def keys(seed: int, layer: int, rows: np.ndarray, samples: np.ndarray) -> np.ndarray:
    """key(layer, r, s) for every global row r (axis 0) and global sample s (axis 1): uint64 [R, S]."""
    h = mix(np.array(seed & MASK64, dtype=U64))
    h = mix(h ^ U64(layer))
    h = mix(h ^ np.asarray(rows, dtype=U64)[:, None])
    return mix(h ^ np.asarray(samples, dtype=U64)[None, :])


def draws(seed: int, layer: int, rows: np.ndarray, samples: np.ndarray, units: int) -> np.ndarray:
    """The 32-bit draws u of units [0, units) of every (global row, global sample): uint32 [R, S, units]."""
    k = keys(seed, layer, rows, samples)
    pairs = np.arange((units + 1) // 2, dtype=U64)
    w = mix(k[:, :, None] ^ pairs[None, None, :])                       # [R, S, pairs]
    lo = (w & U64(0xFFFFFFFF)).astype(np.uint32)
    hi = (w >> U64(32)).astype(np.uint32)
    return np.stack([lo, hi], axis=-1).reshape(k.shape + (2 * pairs.size,))[:, :, :units]


def threshold(p: float) -> int:
    return int(np.rint(np.float64(p) * 2.0 ** 32))


def scale(p: float) -> np.float32:
    return F(0.0) if p >= 1.0 else F(1.0 / np.float64(F(1.0 - np.float64(p))))


def dropped(seed: int, layer: int, rows, samples, units: int, p: float) -> np.ndarray:
    """bool [R, S, units]: the units the head's dropout on layer `layer`'s input drops."""
    return draws(seed, layer, rows, samples, units).astype(np.uint64) < U64(threshold(p)) if p > 0 else \
        np.zeros((len(rows), len(samples), units), dtype=bool)


def dense(x: np.ndarray, kernel: np.ndarray, bias: np.ndarray) -> np.ndarray:
    """x [R, S, in] float32 -> [R, S, out]: ascending units, every product and sum rounded once, then + bias."""
    acc = np.zeros(x.shape[:2] + (kernel.shape[1],), dtype=F)
    for j in range(kernel.shape[0]):
        acc = (acc + (x[:, :, j:j + 1] * kernel[j][None, None, :]).astype(F)).astype(F)
    return (acc + bias.astype(F)).astype(F)


def relu(z: np.ndarray) -> np.ndarray:
    return np.where(z < 0, F(0), z).astype(F)


def preact(h: np.ndarray, layers: Sequence[Tuple[np.ndarray, np.ndarray, float, str]], seed: int, samples: int,
           row0: int = 0, sample0: int = 0) -> np.ndarray:
    """The last layer's pre-activations [rows, samples, C] (float32), as tip_mc_head's TIP_MC_PREACT writes them.
    layers: (kernel [in, out], bias [out], p, activation) as engine.mc_head takes them."""
    h = np.asarray(h, dtype=F)
    rows = np.arange(row0, row0 + h.shape[0])
    smp = np.arange(sample0, sample0 + samples)
    x = np.broadcast_to(h[:, None, :], (h.shape[0], samples, h.shape[1]))
    z = None
    for l, (kernel, bias, p, act) in enumerate(layers):
        if z is not None:
            x = relu(z) if layers[l - 1][3] == "relu" else z
        drop = dropped(seed, l, rows, smp, x.shape[2], p)
        xk = np.where(drop, F(0), (x * scale(p)).astype(F)).astype(F)
        z = dense(xk, np.asarray(kernel, dtype=F), np.asarray(bias, dtype=F))
    return z


def softmax64(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, dtype=np.float64)
    e = np.exp(z - z.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)
