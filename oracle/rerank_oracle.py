"""NumPy reference of the exact re-rank's C contract (tip_nn_rerank, include/b200tip.h) and of the hand-over
steps around it (TEST INFRASTRUCTURE ONLY): the fused next-stage query pack (tip_nn_query_prep's one-segment
operand) and the result scatter of tip_dsa_pack_out.

rerank() states what every output row must hold:
  * a query whose class lies outside [0, n_classes): NaN / -1 / -1 and a zero row, not counted;
  * 1..cap candidate entries: the rows the entries name (mask bit set, 0 <= j < n, j inside the mode's range;
    duplicates allowed) and nothing else;
  * no list, 0 entries or more than cap entries: the whole range, and the query counts in stats[0];
  * distances are the reference's expression np.linalg.norm(x[None, None, :] - t[rows][None], axis=2) in the
    input dtype (surprise.py:638-640); the winner is the minimum of (distance, t_gid) (t_gid: the position);
  * an empty set: NaN / -1.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

SAME_CLASS, OTHER_CLASSES = 0, 1

# Trace widths the re-rank's tests run: every register-resident leaf width (d < 128, d == 128), the first leaf
# programs and the splits around powers of two, up to the widest leaf program (2^23) and one past it (the
# generic recursion).
KERNEL_WIDTHS = (list(range(1, 137)) + [137, 143, 144, 255, 256, 257, 263, 264, 511, 512, 513, 1000, 1024, 1025,
                                        2049, 4097, 8193, 65537, 1 << 23, (1 << 23) + 1])


def norms(x: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """The reference's distances from one query to `rows` (k x d), in their dtype."""
    return np.linalg.norm(x[None, None, :] - rows[None], axis=2)[0]


def in_range(j: np.ndarray, class_off: np.ndarray, cls: int, mode: int) -> np.ndarray:
    """Train positions j inside the range a query of class `cls` searches: its own class (SAME_CLASS) or every
    other class (OTHER_CLASSES)."""
    c0, c1, cn = int(class_off[cls]), int(class_off[cls + 1]), int(class_off[-1])
    if mode == SAME_CLASS:
        return (j >= c0) & (j < c1)
    return (j < cn) & ((j < c0) | (j >= c1))


def listed_rows(entries: np.ndarray, n: int) -> np.ndarray:
    """Positions named by (start, 32-bit mask) entries, in entry and bit order, duplicates kept, out-of-bounds
    rows dropped."""
    out = []
    for start, mask in np.asarray(entries, dtype=np.int64).reshape(-1, 2):
        mask &= 0xFFFFFFFF
        for bit in range(32):
            j = int(start) + bit
            if (mask >> bit) & 1 and 0 <= j < n:
                out.append(j)
    return np.asarray(out, dtype=np.int64)


def winner(dist: np.ndarray, gid: np.ndarray) -> int:
    """Index into (dist, gid) of the minimum distance, ties to the lowest gid (np.argmin's first occurrence when
    gid follows position order)."""
    return int(np.lexsort((gid, dist))[0])


def rerank(q: np.ndarray, t: np.ndarray, class_off, q_class: Optional[np.ndarray], mode: int,
           cand_idx: Optional[np.ndarray] = None, cand_cnt: Optional[np.ndarray] = None, cap: int = 1,
           t_gid: Optional[np.ndarray] = None, q_idx: Optional[np.ndarray] = None) -> Dict[str, np.ndarray]:
    """Expected outputs of tip_nn_rerank.  q: queries (rows q_idx[r] when q_idx is given), t: n x d train rows in
    the same dtype, cand_idx: m x cap x 2 int32 entries, cand_cnt: m counts (None: every query is scanned).
    Returns out_dist, out_pos, out_gid, out_rows, scanned (the stats[0] increment) and queued[m] (the queries
    without a usable list, valid class)."""
    class_off = np.asarray(class_off, dtype=np.int64)
    n_classes = class_off.shape[0] - 1
    n, d = t.shape
    m = q.shape[0] if q_idx is None else len(q_idx)
    gids = np.arange(n, dtype=np.int64) if t_gid is None else np.asarray(t_gid, dtype=np.int64)
    out = {"out_dist": np.full(m, np.nan, dtype=t.dtype), "out_pos": np.full(m, -1, dtype=np.int32),
           "out_gid": np.full(m, -1, dtype=np.int32), "out_rows": np.zeros((m, d), dtype=t.dtype),
           "queued": np.zeros(m, dtype=bool)}
    everything = np.arange(n, dtype=np.int64)
    for r in range(m):
        x = q[r if q_idx is None else int(q_idx[r])]
        cls = 0 if q_class is None else int(q_class[r])
        if cls < 0 or cls >= n_classes:
            continue
        cnt = None if cand_cnt is None else int(cand_cnt[r])
        if cnt is None or cnt < 1 or cnt > cap:
            out["queued"][r] = True
            rows = everything[in_range(everything, class_off, cls, mode)]
        else:
            rows = listed_rows(cand_idx[r, :cnt], n)
            rows = rows[in_range(rows, class_off, cls, mode)]
        if rows.size == 0:
            continue
        dist = norms(x, t[rows])
        k = winner(dist, gids[rows])
        j = int(rows[k])
        out["out_dist"][r], out["out_pos"][r], out["out_gid"][r] = dist[k], j, gids[j]
        out["out_rows"][r] = t[j]
    out["scanned"] = int(out["queued"].sum())
    return out


# ---- NumPy's pairwise summation, vectorised (the order the re-rank implements) -----------------------------------
def _split(n: int) -> int:
    """Where NumPy's pairwise sum splits a block of n > 128 elements: n / 2 rounded down to a multiple of 8."""
    n2 = n // 2
    return n2 - n2 % 8


def _leaves(off: int, n: int, out: list):
    """NumPy's leaves (offset, length <= 128) in left-to-right order; returns the tree as nested pairs."""
    if n <= 128:
        out.append((off, n))
        return len(out) - 1
    n2 = _split(n)
    return (_leaves(off, n2, out), _leaves(off + n2, n - n2, out))


def _leaf_sums(a: np.ndarray, leaves: list) -> np.ndarray:
    """Every leaf's sum as NumPy's leaf loop forms it: n < 8 sequential; else eight stride-8 accumulators, the
    tree ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail in order.  Vectorised over the leaves
    of one length."""
    t = a.dtype.type
    res = np.zeros(len(leaves), dtype=a.dtype)
    offs = np.asarray([o for o, _ in leaves], dtype=np.int64)
    lens = np.asarray([l for _, l in leaves], dtype=np.int64)
    for n in np.unique(lens):
        sel = np.nonzero(lens == n)[0]
        blk = a[offs[sel][:, None] + np.arange(n)[None, :]]
        if n < 8:
            s = np.zeros(sel.size, dtype=a.dtype)
            for i in range(n):
                s = s + blk[:, i]
        else:
            lim = n - n % 8
            r = blk[:, :8].copy()
            for i in range(8, lim, 8):
                r = r + blk[:, i:i + 8]
            s = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            for i in range(lim, n):
                s = s + blk[:, i]
        res[sel] = s.astype(t)
    return res


def pairwise_sum(a: np.ndarray):
    """np.add.reduce(a) of a contiguous 1-D float32 / float64 array, restated: the same bits, any length."""
    leaves = []
    tree = _leaves(0, a.shape[0], leaves)
    sums = _leaf_sums(a, leaves)

    def fold(node):
        if isinstance(node, tuple):
            return a.dtype.type(fold(node[0]) + fold(node[1]))
        return sums[node]

    return fold(tree)


def norm_model(x: np.ndarray, y: np.ndarray):
    """sqrt(pairwise_sum((x - y)^2)) in the input dtype: the re-rank's distance, built from its parts."""
    diff = x - y
    return np.sqrt(pairwise_sum(diff * diff))


# ---- the fused next-stage query pack (tip_nn_query_prep, one segment) --------------------------------------------
def pair_pitch(d: int) -> int:
    """tip_pair_pitch(d, 1): the width rounded up to 16, a 16-column tail, rounded up to 64."""
    d16 = (d + 15) & ~15
    return (d16 + 16 + 63) & ~63


def pack_query(rows: np.ndarray, center: Optional[np.ndarray]) -> np.ndarray:
    """The bf16 bits (uint16, rows x pair_pitch(d)) of the packed queries: fl32(x - c) (float64 traces: the
    difference in double, rounded once), bf16 round-to-nearest-even, zeros up to the next multiple of 16, then the
    tail [1, 1, 1, 0, ...]."""
    import torch

    m, d = rows.shape
    c = np.zeros(d, dtype=np.float32) if center is None else np.asarray(center, dtype=np.float32)
    if rows.dtype == np.float64:
        v = (rows - c.astype(np.float64)).astype(np.float32)
    else:
        v = rows.astype(np.float32) - c
    d16 = (d + 15) & ~15
    full = np.zeros((m, pair_pitch(d)), dtype=np.float32)
    full[:, :d] = v
    full[:, d16:d16 + 3] = 1.0
    return torch.from_numpy(full).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def bf16_values(bits: np.ndarray) -> np.ndarray:
    """bf16 bit patterns -> float64 values (exact)."""
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


# ---- tip_dsa_pack_out ----------------------------------------------------------------------------------------
def pack_out(dist_a: np.ndarray, dist_b: np.ndarray, gid: np.ndarray, idx: Optional[np.ndarray], n_total: int,
             out: np.ndarray) -> np.ndarray:
    """out (4 x n_total float64, updated in place and returned): column j = idx[i] (i itself without idx) receives
    dist_a, dist_b, gid and dist_a / dist_b divided in the distances' dtype (surprise.py:595); indices outside
    [0, n_total) are skipped."""
    for i in range(dist_a.shape[0]):
        j = i if idx is None else int(idx[i])
        if not 0 <= j < n_total:
            continue
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            ratio = dist_a[i] / dist_b[i]
        out[:, j] = (dist_a[i], dist_b[i], gid[i], ratio)
    return out
