"""float64 references of the LSA kernels (tip_pair_prep / tip_pair_prep_f16 -> tip_kde_lse / tip_kde_lse_f16 ->
tip_kde_combine, and tip_whiten / tip_row_sqnorm) (TEST INFRASTRUCTURE ONLY).

Written from the operand layout and the error model that include/b200tip.h and DESIGN.md §4 / §5 document, not from
the CUDA:

  * `pack_lse` / `pack_f16`   the three-segment split-bf16 and the one-segment fp16 operands with LSA's arguments;
  * `lse_parts`               per-(slot, row) (max_j a_ij, sum_j exp(a_ij - max)) of a work list, with a formed from
                              the packed operands themselves (operand rounding is not kernel error), and `lse_bound`,
                              the kernel's error budget for each partial in the log domain;
  * `int_lse_operands` / `exact_lse_parts`   the exact construction below and its integer partials;
  * `check_kde_work_list`     what the pass needs of a work list over one query block x one column range;
  * `combine_ref`             the float64 merge of the partials with the budget of tip_kde_combine, and
                              `combine_unit_replica`, its fp32 order restated for partials whose maxima are 0 or -inf;
  * `whiten_bound`            (x[:, cols] - mu) . w in float64 with the budget of the fp32 FMA chain.

Exact construction of the log-sum-exp pass.  Training rows are p_j = 16 e_k(j) or 0, query rows q in {0, 8}^d.  Every
operand is bf16- and fp16-exact, the low parts are 0, and the norm term -|p|^2 / 2 in {0, -128} splits exactly
(fp16: -2 at the tail scale S = 64, against a query tail of 64).  So a_ij = 128 [q_i,k(j) = 8] - 128 for p_j != 0 and
a_ij = 0 for p_j = 0: every product and partial sum of the K-loop is an integer of magnitude <= 128, and a is exactly
0 ("hit") or -128 ("miss") in any summation order.  In a span with a hit the kernel's rescale factor
ex2.approx(-128 log2 e) and every miss term lie below fp32's range and flush to exactly 0 (.ftz), so part_max = 0 and
part_sum is the integer number of hit columns; a span without a hit gives part_max = -128 and part_sum = its width (the
offset fl(128 log2 e) is exact, so each term is ex2.approx(0)).  A missing, duplicated or foreign column changes such a
count by 1; the comparison allows 2^-20 of the count (the documented 2-ulp error of ex2.approx, which would matter
only if ex2.approx(0) were not exactly 1).  Columns past the end of the training matrix come out of TMA as zeros
(a = 0: hits), so a missing col1 mask is visible too.

Inputs are NumPy arrays (the float64 partials also take a torch device to run on); nothing in the product package
imports this module.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from .sil_oracle import bf16_bits, bf16_rn, pair_pitch, split3

EPS = 2.0 ** -24            # unit roundoff of fp32
EXACT_RTOL = 2.0 ** -20     # exact construction: |part_sum - count| <= EXACT_RTOL * count
F16_MAX = 65504.0
F16_NORM_SCALE = 64.0       # engine.F16_NORM_SCALE
HIT, MISS = 0.0, -128.0     # the two values of a in the exact construction
ROW_TILE, COL_TILE = 128, 256


def pair_pitch1(d: int) -> int:
    """row pitch of the one-segment operand in elements: d16 + a 16-wide tail, rounded up to 64"""
    d16 = -(-d // 16) * 16
    return (d16 + 16 + 63) // 64 * 64


def _centred(x: np.ndarray, center: Optional[np.ndarray]) -> np.ndarray:
    """v = fl32(x - c): one fp32 subtraction for float32 rows, the double difference rounded once for float64"""
    x = np.asarray(x)
    assert x.dtype in (np.float32, np.float64) and x.ndim == 2
    c = np.zeros(x.shape[1], dtype=np.float32) if center is None else np.asarray(center, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        return (x - c) if x.dtype == np.float32 else (x - c.astype(np.float64)).astype(np.float32)


def _sqnorm(v: np.ndarray) -> np.ndarray:
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sum(v.astype(np.float64) ** 2, axis=1).astype(np.float32)


# ---- operand packing -------------------------------------------------------------------------------------------
def lse_tail(sqnorm: np.ndarray) -> np.ndarray:
    """train tail of the three-segment operand: split3(fl32(-0.5 * sqnorm)) as float32 [rows, 3]"""
    return split3(np.float32(-0.5) * np.asarray(sqnorm, dtype=np.float32))


def pack_lse(x: np.ndarray, role: str, center: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """NumPy emulation of tip_pair_prep(segments=3) with LSA's arguments (scale 1; train: norm_coef -0.5).  Returns
    (pack as uint16 bf16 bit patterns [n, tip_pair_pitch(d, 3)], sqnorm float32 [n] = fp32 of the double sum v^2):
      query row [h | l | h | 1, 1, 1, 0...], train row [h | h | l | split3(-|v|^2 / 2) | 0...],
      v = fl32(x - c), h = bf16(v), l = bf16(v - h), each segment zero-padded from d to d16.  Finite rows only."""
    assert role in ("query", "train")
    v = _centred(x, center)
    n, d = v.shape
    d16 = -(-d // 16) * 16
    vp = np.zeros((n, d16), dtype=np.float32)
    vp[:, :d] = v
    h = bf16_rn(vp)
    lo = bf16_rn(vp - h)                  # v - h is exact in fp32
    sq = _sqnorm(v)
    out = np.zeros((n, pair_pitch(d)), dtype=np.float32)
    if role == "query":
        out[:, :d16], out[:, d16:2 * d16], out[:, 2 * d16:3 * d16] = h, lo, h
        out[:, 3 * d16:3 * d16 + 3] = 1.0
    else:
        out[:, :d16], out[:, d16:2 * d16], out[:, 2 * d16:3 * d16] = h, h, lo
        out[:, 3 * d16:3 * d16 + 3] = lse_tail(sq)
    return bf16_bits(out), sq


def _f16(v: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(v, dtype=np.float32).astype(np.float16)


def f16_tail(sqnorm: np.ndarray, norm_coef: float, S: float) -> Tuple[np.ndarray, np.ndarray]:
    """train tail of the fp16 operand: the 3-way fp16 split of cv = fl32(fl32(norm_coef * sqnorm) / S) as float16
    [rows, 3], and whether cv is out of fp16's finite range"""
    with np.errstate(over="ignore", invalid="ignore"):
        cv = (np.float32(norm_coef) * np.asarray(sqnorm, dtype=np.float32)) / np.float32(S)
        c0 = _f16(cv).astype(np.float32)
        c1 = _f16(cv - c0).astype(np.float32)
        c2 = _f16((cv - c0) - c1)
    return np.stack([c0.astype(np.float16), c1.astype(np.float16), c2], axis=-1), ~(np.abs(cv) <= F16_MAX)


def pack_f16(x: np.ndarray, role: str, norm_coef: float, S: float,
             center: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, bool]:
    """NumPy emulation of tip_pair_prep_f16.  Returns (pack as uint16 fp16 bit patterns [n, tip_pair_pitch(d, 1)],
    sqnorm float32 [n], flag): row [fp16_rn(v) | tail | 0...], v = fl32(x - c) zero-padded to d16; query tail
    [S, S, S], train tail f16_tail(|v|^2); flag = some |v| is not <= 65504 (inf, NaN) or, for the train role, some
    norm term cv is not."""
    assert role in ("query", "train")
    v = _centred(x, center)
    n, d = v.shape
    d16 = -(-d // 16) * 16
    sq = _sqnorm(v)
    out = np.zeros((n, pair_pitch1(d)), dtype=np.float16)
    out[:, :d] = _f16(v)
    flag = bool(np.any(~(np.abs(v) <= F16_MAX)))
    if role == "query":
        out[:, d16:d16 + 3] = np.float16(S)
    else:
        tail, bad = f16_tail(sq, norm_coef, S)
        out[:, d16:d16 + 3] = tail
        flag |= bool(np.any(bad))
    return out.view(np.uint16), sq, flag


def decode(bits: np.ndarray, kind: str) -> np.ndarray:
    """float64 values of packed bf16 ("bf16") or fp16 ("f16") bit patterns"""
    bits = np.asarray(bits, dtype=np.uint16)
    if kind == "bf16":
        return (bits.astype(np.uint32) << np.uint32(16)).view(np.float32).astype(np.float64)
    assert kind == "f16"
    return bits.view(np.float16).astype(np.float64)


def k_width(d: int, kind: str) -> int:
    """packed width K the kernel's K-loop runs over (tail block included)"""
    d16 = -(-d // 16) * 16
    return (3 if kind == "bf16" else 1) * d16 + 16


# ---- float64 partials ------------------------------------------------------------------------------------------
def _spans(items: np.ndarray, m: int):
    """{(col0, col1, slot): rows covered} of a work list"""
    spans = {}
    for q0, qr, c0, c1, slot, _ in np.asarray(items).tolist():
        if c1 <= c0:
            continue
        rows = spans.setdefault((c0, c1, slot), np.zeros(m, dtype=bool))
        rows[q0:q0 + qr] = True
    return spans


def lse_parts(q_pack, t_pack, items: np.ndarray, slots: int, m: int, kind: str = "bf16", device=None,
              stats: bool = False):
    """float64 partials of tip_kde_lse (kind "bf16") / tip_kde_lse_f16 ("f16") for a work list: a = decode(q_pack) @
    decode(t_pack).T over each item's span; part_max[slot, row] = max_j a, part_sum = sum_j exp(a - part_max); NaN
    where no item writes.  Returns (part_max, part_sum, covered) and, with stats=True, a dict of per-(slot, row) inputs
    of lse_bound: absdot = max_j sum_k |q_k t_k|, amax = max_j |a_j|, wdist = sum_j w_j (max - a_j) / sum_j w_j with
    w_j = exp(a_j - max), width = span width.  Runs in torch float64 on `device` (default: CPU)."""
    import torch

    pm = np.full((slots, m), np.nan)
    ps = np.full((slots, m), np.nan)
    covered = np.zeros((slots, m), dtype=bool)
    st = {k: np.full((slots, m), np.nan) for k in ("absdot", "amax", "wdist", "width")}
    spans = _spans(items, m)
    if not spans:
        return (pm, ps, covered, st) if stats else (pm, ps, covered)
    q = torch.as_tensor(decode(q_pack, kind), device=device)
    t = torch.as_tensor(decode(t_pack, kind), device=device)
    idx = lambda a: torch.as_tensor(a, dtype=torch.int64, device=q.device)
    for (c0, c1, slot), mask in spans.items():
        rows = np.flatnonzero(mask)
        qr, tc = q[idx(rows)], t[c0:c1]
        a = qr @ tc.T
        mx = a.max(dim=1).values
        w = torch.exp(a - mx[:, None])
        sw = w.sum(1)
        pm[slot, rows], ps[slot, rows] = mx.cpu().numpy(), sw.cpu().numpy()
        covered[slot, rows] = True
        if stats:
            st["absdot"][slot, rows] = (qr.abs() @ tc.abs().T).max(dim=1).values.cpu().numpy()
            st["amax"][slot, rows] = a.abs().max(dim=1).values.cpu().numpy()
            st["wdist"][slot, rows] = ((w * (mx[:, None] - a)).sum(1) / sw).cpu().numpy()
            st["width"][slot, rows] = c1 - c0
    return (pm, ps, covered, st) if stats else (pm, ps, covered)


def lse_bound(st: dict, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """(bound on |part_max - max|, bound on |part_max + log part_sum - logsumexp|) per (slot, row), natural-log units,
    for a K-loop of packed width k (k_width).  Per term of a span (eps = 2^-24):
      * the fp32 accumulation of the k products and the tail, nothing better than truncating adds (DESIGN.md §4):
        E = (k + 16) 2^-23 sum_k |q_k t_k|; it moves the max and every term by at most E;
      * the offset fl(-run_max log2 e) (eps |run_max| <= eps (amax + E)) and the fma's rounding and fp32 log2 e
        (2 eps |a_j - run_max| <= 2 eps (max - a_j + 2E): weighted by the terms, 2 eps (wdist + 2E));
      * ex2.approx, 2^-22 relative, per term and per rescale (at most one rescale per 32-column chunk), each rescale
        also rounding its product (eps) and its argument (the arguments sum to at most the span's range, 2 amax);
      * the fp32 sum: a depth-5 tree per chunk, then one add per chunk;
      * terms and rescaled sums below 2^-126 flush to 0: at most 2 width 2^-126 of the sum (whose largest term is 1).
    A relative error r of the sum is r (1 + r) in the log; the 1.01 covers that and the other second-order terms."""
    e = (k + 16) * 2.0 ** -23 * st["absdot"]
    chunks = np.ceil(st["width"] / 32.0)
    lse = (e + EPS * (st["amax"] + e) + 2 * EPS * (st["wdist"] + 2 * e) + 4 * EPS + chunks * 5 * EPS
           + 2 * EPS * st["amax"] + (5 + chunks) * EPS + 2 * st["width"] * 2.0 ** -126)
    return e, lse * 1.01


def lse_excess(part_max, part_sum, ref_max, ref_sum, st: dict, k: int) -> Tuple[float, float]:
    """worst |err| / bound of part_max and of part_max + log part_sum over the covered entries (inf for a
    non-finite device value)"""
    cov = ~np.isnan(ref_max)
    pmx, psm = np.asarray(part_max, np.float64)[cov], np.asarray(part_sum, np.float64)[cov]
    if not (np.all(np.isfinite(pmx)) and np.all(psm > 0) and np.all(np.isfinite(psm))):
        return np.inf, np.inf
    bm, bl = lse_bound({kk: v[cov] for kk, v in st.items()}, k)
    em = np.abs(pmx - ref_max[cov]) / bm
    el = np.abs((pmx + np.log(psm)) - (ref_max[cov] + np.log(ref_sum[cov]))) / bl
    return float(em.max(initial=0.0)), float(el.max(initial=0.0))


# ---- the exact construction ------------------------------------------------------------------------------------
def int_lse_operands(m: int, n: int, d: int, seed: int, zero_frac: float = 0.02) -> Tuple[np.ndarray, np.ndarray]:
    """(q [m, d], p [n, d]) float64 of the exact construction.  p_j = 16 e_k(j); the first min(n, d) columns take
    distinct coordinates and the last one takes d - 1, so every 16-wide K step is used, the last partial one too;
    a zero_frac share of the columns in the first half are zero rows (always hits), the second half has none.  Query
    rows cycle through four kinds: one coordinate set (hits are rare: spans with and without a hit), dense random bits,
    all zero (hits only on zero columns) and about four coordinates set."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, d, size=n)
    first = min(n, d)
    k[:first] = rng.permutation(d)[:first]
    k[-1] = d - 1
    p = np.zeros((n, d))
    p[np.arange(n), k] = 16.0
    half = n // 2
    if half > 0:
        zero = rng.choice(half, size=int(round(zero_frac * half)), replace=False)
        p[zero] = 0.0
    q = np.zeros((m, d))
    for r in range(m):
        kind = r % 4
        if kind == 0:
            q[r, rng.integers(0, d)] = 8.0
        elif kind == 1:
            q[r] = 8.0 * (rng.random(d) < 0.5)
        elif kind == 3:
            q[r] = 8.0 * (rng.random(d) < min(1.0, 4.0 / d))
    return q, p


def hit_prefix(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """int32 [m, n + 1]: number of hit columns (a = 0) of each query row among columns [0, j)"""
    zero = ~np.any(p != 0, axis=1)
    k = np.argmax(p != 0, axis=1)
    hits = zero[None, :] | (q != 0)[:, k]
    out = np.zeros((q.shape[0], p.shape[0] + 1), dtype=np.int32)
    np.cumsum(hits, axis=1, out=out[:, 1:])
    return out


def exact_lse_parts(prefix: np.ndarray, items: np.ndarray, slots: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """what the kernel must write on the exact construction (hit_prefix of it): part_max 0 and part_sum = hit count
    for a span with a hit, -128 and the span width for one without; NaN where no item writes; and the covered mask"""
    m = prefix.shape[0]
    pm = np.full((slots, m), np.nan)
    ps = np.full((slots, m), np.nan)
    for (c0, c1, slot), mask in _spans(items, m).items():
        hits = (prefix[mask, c1] - prefix[mask, c0]).astype(np.float64)
        pm[slot, mask] = np.where(hits > 0, HIT, MISS)
        ps[slot, mask] = np.where(hits > 0, hits, float(c1 - c0))
    return pm, ps, ~np.isnan(pm)


def exact_excess(part_max, part_sum, ref_max, ref_sum) -> float:
    """worst |part_sum - count| / (EXACT_RTOL count) over the covered entries; inf if a covered part_max differs, a
    covered entry is not finite or an uncovered entry was written (device outputs start as NaN)"""
    part_max = np.asarray(part_max, dtype=np.float64)
    part_sum = np.asarray(part_sum, dtype=np.float64)
    cov = ~np.isnan(ref_max)
    if not np.all(np.isnan(part_max[~cov]) & np.isnan(part_sum[~cov])):
        return np.inf
    if not (np.all(np.isfinite(part_max[cov])) and np.all(np.isfinite(part_sum[cov]))):
        return np.inf
    if not np.array_equal(part_max[cov], ref_max[cov]):
        return np.inf
    err = np.abs(part_sum[cov] - ref_sum[cov]) / (EXACT_RTOL * ref_sum[cov])
    return float(err.max(initial=0.0))


# ---- work lists ------------------------------------------------------------------------------------------------
def check_kde_work_list(items: np.ndarray, m: int, n: int, span_tiles: int, row_tile: int = ROW_TILE,
                        col_tile: int = COL_TILE) -> None:
    """Asserts what the log-sum-exp pass needs of a work list over one query block [0, m) x one column range [0, n),
    independently of how it was built (the partials above follow whatever list they are given): query tiles start
    every row_tile rows and hold min(row_tile, m - q_row0) rows; each tile's spans cover [0, n) exactly once, are
    non-empty, at most span_tiles * col_tile wide and end at or before n; the spans of one tile have distinct slots."""
    items = np.asarray(items, dtype=np.int64)
    assert items.ndim == 2 and items.shape[1] == 6
    q0, qr, c0, c1, slot = (items[:, i] for i in range(5))
    assert np.all(q0 % row_tile == 0) and np.all((q0 >= 0) & (q0 < m)), "query tiles"
    assert np.array_equal(qr, np.minimum(row_tile, m - q0)), "q_rows of a tile"
    assert np.all((c0 >= 0) & (c0 < c1) & (c1 <= n)), "span bounds"
    assert np.all(c1 - c0 <= span_tiles * col_tile), "span wider than span_tiles * col_tile"
    assert np.all(slot >= 0), "slot"
    assert set(q0.tolist()) == set(range(0, m, row_tile)), "a query tile is missing"
    for t in range(0, m, row_tile):
        mine = items[q0 == t]
        sp = sorted(zip(mine[:, 2].tolist(), mine[:, 3].tolist()))
        assert [a for a, _ in sp] == [0] + [b for _, b in sp[:-1]] and sp[-1][1] == n, f"tile {t}: spans {sp[:8]}"
        assert np.unique(mine[:, 4]).shape[0] == mine.shape[0], f"tile {t}: two spans share a slot"


def residency_order(items: np.ndarray, g: int) -> np.ndarray:
    """The list reordered for a persistent grid of g CTAs (CTA b runs items b, b + g, ...) so that each CTA runs one
    contiguous piece of the query-tile-major order: items w and w + g mostly share a query tile, which the
    resident-query kernel then keeps in shared memory.  Longer pieces go to the first CTAs, so every round but the
    last is full and no padding item is needed."""
    items = np.asarray(items)
    srt = items[np.lexsort((items[:, 2], items[:, 0]))]
    k = srt.shape[0]
    g = min(g, k)
    sizes = [k // g + (1 if b < k % g else 0) for b in range(g)]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    out = np.empty_like(srt)
    for b in range(g):
        for r in range(sizes[b]):
            out[r * g + b] = srt[starts[b] + r]
    return out


def resident_pairs(items: np.ndarray, g: int) -> int:
    """number of w with items w and w + g on one query tile: consecutive items of one CTA that reuse its query tile"""
    items = np.asarray(items)
    g = min(g, items.shape[0])
    return int(np.sum(items[:-g, 0] == items[g:, 0])) if items.shape[0] > g else 0


def ragged_items(m: int, n: int, span_tiles: int, seed: int, row_tile: int = ROW_TILE,
                 col_tile: int = COL_TILE) -> np.ndarray:
    """A valid list whose spans have random widths (1 .. span_tiles * col_tile columns): span ends fall inside
    128-column tiles next to real training rows, so that a missing col1 mask takes in columns of the next span"""
    rng = np.random.default_rng(seed)
    out = []
    for q0 in range(0, m, row_tile):
        c0, s = 0, 0
        while c0 < n:
            c1 = min(n, c0 + int(rng.integers(1, span_tiles * col_tile + 1)))
            out.append((q0, min(row_tile, m - q0), c0, c1, s, 0))
            c0, s = c1, s + 1
    return np.asarray(out, dtype=np.int32)


# ---- the merge of the partials ---------------------------------------------------------------------------------
def combine_ref(part_max: np.ndarray, part_sum: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """float64 merge of [slots, m] partials: M = max over the slots whose max is > -inf (NaN and -inf slots are
    skipped), S = sum ps exp(pm - M); (-inf, 0) for a row without such a slot.  Returns (M, S, bound on |S_dev - S|).
    tip_kde_combine merges slot s into group s mod 8 online (rescale by expf(old - new) when the max rises, else
    add ps expf(pm - max)), then the 8 groups into the row.  So a slot's term passes through at most
    ceil(slots / 8) + 1 expf-and-multiply steps (expf 2 ulp = 4 eps, the product eps) whose arguments, each rounded
    (eps relative), sum to M - pm; and through at most ceil(slots / 8) + 8 fp32 adds.  Values below 2^-126 may flush."""
    pm = np.asarray(part_max, dtype=np.float32).astype(np.float64)
    ps = np.asarray(part_sum, dtype=np.float32).astype(np.float64)
    slots = pm.shape[0]
    live = pm > -np.inf
    M = np.where(live, pm, -np.inf).max(axis=0)
    some = np.isfinite(M)
    with np.errstate(invalid="ignore", over="ignore"):
        t = np.where(live, ps * np.exp(np.where(live, pm, 0.0) - np.where(some, M, 0.0)), 0.0)
        dist = np.where(live, np.where(some, M, 0.0) - np.where(live, pm, 0.0), 0.0)
    S = t.sum(axis=0)
    ng = -(-slots // 8)
    per = ((ng + 1) * 5 + ng + 8) * EPS
    bound = (np.abs(t) * (per + EPS * dist)).sum(axis=0) * 1.01
    bound += 2 * slots * 2.0 ** -126 * np.where(live, np.abs(ps), 0.0).max(axis=0, initial=0.0)
    return M, np.where(some, S, 0.0), np.where(some, bound, 0.0)


def combine_unit_replica(part_max: np.ndarray, part_sum: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """tip_kde_combine restated in fp32 for partials whose maxima are all 0 or -inf, where every factor is expf(0) = 1
    or expf(-inf) = 0 and only the order of the fp32 adds is left: per row, group g = slots g, g + 8, ... summed from 0
    in ascending slot order, then the groups with a finite max summed from 0 in ascending g"""
    pm = np.asarray(part_max, dtype=np.float32)
    ps = np.asarray(part_sum, dtype=np.float32)
    assert np.all((pm == 0) | (pm == -np.inf))
    slots, m = pm.shape
    gsum = np.zeros((8, m), dtype=np.float32)
    glive = np.zeros((8, m), dtype=bool)
    for s in range(slots):
        live = pm[s] == 0
        gsum[s % 8] = np.where(live, gsum[s % 8] + ps[s], gsum[s % 8])
        glive[s % 8] |= live
    S = np.zeros(m, dtype=np.float32)
    for g in range(8):
        S = np.where(glive[g], S + gsum[g], S)
    M = np.where(glive.any(axis=0), np.float32(0), np.float32(-np.inf))
    return M, S


# ---- whitening -------------------------------------------------------------------------------------------------
def whiten_bound(x: np.ndarray, cols: Optional[np.ndarray], mu: np.ndarray, w: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """float64 (x[:, cols] - mu) . w (cols None: the first d_out columns) and the budget of tip_whiten: v = x - mu is
    formed in double and rounded to fp32 once (eps |v|), then each output is a sequential fp32 FMA chain over d_out
    terms (gamma_dn = dn eps / (1 - dn eps) of sum_k |v_k w_kj|); gradual underflow adds 2^-149 per step."""
    x = np.asarray(x)
    dn = w.shape[0]
    xs = (x[:, np.asarray(cols)] if cols is not None else x[:, :dn]).astype(np.float64)
    v = xs - np.asarray(mu, dtype=np.float64)
    w64 = np.asarray(w, dtype=np.float32).astype(np.float64)
    ref = v @ w64
    gamma = dn * EPS / (1 - dn * EPS)
    bound = ((gamma + EPS) * (np.abs(v) @ np.abs(w64))) * 1.001 + dn * 2.0 ** -149
    return ref, bound
