"""Float64 model of one tip_nn_filter call (csrc/pair_tc.cu, pair_kernel<MODE_NN, ...>) on the exact buffers the kernel
read and wrote (TEST INFRASTRUCTURE ONLY: plain NumPy, torch only for bf16 rounding; it never imports the extension).

DSA's exactness (DESIGN.md §4) rests on two properties of the filter's outputs, which end-to-end tests see only when
a lost column happens to be NumPy's argmin:

1. the shared row minimum: row_min_bits[i] is max(min_{j in R_i} acc_ij + |x_b|^2, 0), within the accumulation slack;
2. complete candidate lists: every column inside the final window appears in some mask.

check() tests both, and that every list is well formed and every admitted column sound, on
  * the accumulators a = Q_b . T_b^T over the whole packed width (tail block included), from the packed bf16 rows;
  * the per-row window constants nx, r, e2, g as the kernel computes them in float32;
  * the two threshold bounds threshold_lo / threshold_hi around nn_threshold();
  * each row's range R_i: the union of the item spans covering row i, minus its own class for flagged items.
It returns findings (row, column, item, value, bound) rather than asserting, so that a failure points at its cause.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

F32 = np.float32
INF_BITS = 0x7F800000
CHUNK = 32


def _bf16(a: np.ndarray) -> np.ndarray:
    """Round to bfloat16 (nearest even) and back to float32, through torch."""
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(torch.bfloat16).to(torch.float32).numpy()


def threshold_lo(s, nx, e2, g):
    """nn_threshold() of csrc/pair_tc.cu in float32, with sqrt.approx modelled 2 ulp LOW (worst case), never above
    the kernel's value: fmaf(r, r, g) is one rounding, which two roundings (r * r, then + g) can overshoot by an ulp
    of r^2 + g, and thr + |thr| 1e-6 may or may not be contracted; each is taken at its lower end."""
    root = F32(np.sqrt(F32(s + g), dtype=F32)) * F32(1.0 - 2.0 ** -22)
    r = F32(F32(root + e2) * F32(1.00004))
    rr = np.nextafter(F32(np.float64(r) * np.float64(r) + np.float64(g)), F32(-np.inf))
    thr = F32(rr - nx)
    tail = min(F32(thr + F32(abs(thr)) * F32(1e-6)),
               np.nextafter(F32(np.float64(thr) + np.float64(abs(thr)) * np.float64(F32(1e-6))), F32(-np.inf)))
    return F32(tail + F32(1e-30))


def threshold_hi(s, nx, e2, g):
    """nn_threshold() of csrc/pair_tc.cu at its widest: sqrt.approx 2 ulp high, every float32 rounding against us
    (the kernel's 1e-30f is float32's nearest value, slightly above 1e-30)."""
    root = np.sqrt(s + g) * (1 + 2.0 ** -21)
    r = (root + e2) * 1.00004 * (1 + 2.0 ** -22)
    thr = r * r + g - nx
    return thr + abs(thr) * 1e-6 + float(F32(1e-30)) + 2.0 ** -20 * (abs(nx) + r * r)


def bf16_bits(u16: np.ndarray) -> np.ndarray:
    """bfloat16 bit patterns (uint16) -> their float64 values."""
    return (np.asarray(u16, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def k16_of(d: int) -> int:
    """K16 steps of a one-segment packed row of width d: round_up(d, 16) + the 16-wide tail block."""
    return ((d + 15) // 16 * 16 + 16) // 16


def accumulators(q_pack: np.ndarray, t_pack: np.ndarray, d: int):
    """a[i, j] = <Q_b[i], T_b[j]> over the packed width the kernel multiplies (k16 * 16 columns, tail included), in
    float64, and a bound on its float64 summation error.  Every bf16 x bf16 product is exact in float64 (8 + 8
    significand bits), so the only error is the summation's: whatever the order, |fl(sum) - sum| <= (K - 1) u sum|p|
    / (1 - (K - 1) u) with u = 2^-53 (Higham, Accuracy and Stability of Numerical Algorithms, (3.4)); K 2^-53 sum|p|
    is above it for every K here."""
    k = 16 * k16_of(d)
    q = bf16_bits(q_pack)[:, :k]
    t = bf16_bits(t_pack)[:, :k]
    a = q @ t.T
    slack = (k * 2.0 ** -53) * (np.abs(q) @ np.abs(t).T)
    return a, slack


@dataclass
class Window:
    """Per-row constants of the kernel's window, float32, as pair_kernel computes them (lines around `s.e2 =`) from
    tip_nn_filter's gamma / eps2.  e2 is bracketed [e2_lo, e2_hi] by one ulp on each side of both the fused and the
    unfused evaluation of (q_err + t_err) + 1.2e-7 r, since nvcc may contract it."""
    nx: np.ndarray
    r: np.ndarray
    e2_lo: np.ndarray
    e2_hi: np.ndarray
    g: np.ndarray


def window(q_sqnorm: np.ndarray, q_rounderr: Optional[np.ndarray], t_rmax: float, t_errmax: float, d: int) -> Window:
    nx = np.asarray(q_sqnorm, dtype=F32)
    r = (np.sqrt(nx, dtype=F32) + F32(t_rmax)).astype(F32)
    gamma = F32(F32(16 * k16_of(d) + 16) * F32(1.1920929e-7))
    g = ((gamma * r).astype(F32) * r).astype(F32)
    if q_rounderr is None:
        e2 = (F32(F32(2.0) * F32(1.96e-3)) * r).astype(F32)           # the a-priori bound 2 eps' r
        return Window(nx, r, e2, e2, g)
    u = (np.asarray(q_rounderr, dtype=F32) + F32(t_errmax)).astype(F32)
    v = [(u + (F32(1.2e-7) * r).astype(F32)).astype(F32),
         (u.astype(np.float64) + np.float64(F32(1.2e-7)) * r.astype(np.float64)).astype(F32)]
    e2 = [((F32(2.0) * vv).astype(F32) * F32(1.00001)).astype(F32) for vv in v]
    return Window(nx, r, np.nextafter(np.minimum(*e2), F32(0)), np.nextafter(np.maximum(*e2), F32(np.inf)), g)


def row_ranges(m: int, n: int, items: np.ndarray, q_class: Optional[np.ndarray] = None,
               class_off: Optional[np.ndarray] = None):
    """R_i as an m x n mask, the item that scans each (row, column) pair (-1: none) and how many items scan it.
    Item w covers rows [q_row0, q_row0 + q_rows) and columns [col0, col1); with flag bit 0 (and q_class / class_off
    passed to the kernel) a row of class c skips [class_off[c], class_off[c + 1])."""
    inr = np.zeros((m, n), dtype=bool)
    owner = np.full((m, n), -1, dtype=np.int32)
    times = np.zeros((m, n), dtype=np.int16)
    cols = np.arange(n)
    excl = q_class is not None and class_off is not None
    for w, (r0, nr, c0, c1, _slot, flag) in enumerate(np.asarray(items, dtype=np.int64).reshape(-1, 6)):
        i0, i1 = max(int(r0), 0), min(int(r0 + nr), m)
        if c1 <= c0 or i1 <= i0:
            continue
        cov = np.broadcast_to((cols >= c0) & (cols < c1), (i1 - i0, n))
        if excl and (flag & 1):
            c = np.asarray(q_class[i0:i1], dtype=np.int64)
            lo, hi = np.asarray(class_off, dtype=np.int64)[c], np.asarray(class_off, dtype=np.int64)[c + 1]
            cov = cov & ~((cols >= lo[:, None]) & (cols < hi[:, None]))
        inr[i0:i1] |= cov
        owner[i0:i1][cov] = w
        times[i0:i1] += cov
    return inr, owner, times


@dataclass
class Report:
    findings: List[dict] = field(default_factory=list)
    rowmin_frac: float = 0.0         # worst |row_min - expected| / bound over the rows with a non-empty range
    required_extra: int = 0          # (row, column) pairs completeness required beyond each row's argmin
    outside: int = 0                 # in-range columns of admitted chunks outside their chunk's widest window
    overflowed: int = 0              # rows with cnt > cap (only their first cap entries are checked)
    checked_rows: int = 0

    def add(self, kind, row, col=-1, item=-1, value=float("nan"), bound=float("nan")):
        self.findings.append(dict(kind=kind, row=int(row), col=int(col), item=int(item), value=float(value),
                                  bound=float(bound)))

    def summary(self, limit: int = 12) -> str:
        return "\n".join(f"{f['kind']}: row {f['row']} col {f['col']} item {f['item']} value {f['value']!r} "
                         f"bound {f['bound']!r}" for f in self.findings[:limit]) + \
            (f"\n... {len(self.findings)} findings" if len(self.findings) > limit else "")


def check(a: np.ndarray, slack: np.ndarray, win: Window, inr: np.ndarray, owner: np.ndarray, row_min_bits: np.ndarray,
          cand_idx: np.ndarray, cand_cnt: np.ndarray, cap: int, seed_bits: Optional[np.ndarray] = None,
          times: Optional[np.ndarray] = None) -> Report:
    """Check one filter call's outputs against the model.  a, slack: accumulators(); win: window(); inr, owner,
    times: row_ranges(); row_min_bits (uint32), cand_idx (m x cap x 2 int32), cand_cnt: the kernel's outputs;
    seed_bits: the row_min_bits the call started from (None: +inf, tip_nn_query_prep's state).

    Row minimum.  With mu_i = min_{j in R_i} a_ij the kernel's fp32 accumulators differ from a by at most g_i, so
    the smallest of them, mu'_i, is within g_i of mu_i.  It is inside every threshold the row passes through
    (nn_threshold(max(v + nx, 0)) >= v, and every running minimum comes from some value >= mu'_i or from the seed),
    so row_min = min(S_i, max(mu'_i + nx_i, 0)) in float32: |row_min - min(S_i, max(mu_i + nx_i, 0))| <= g_i +
    2^-22 (|mu_i| + nx_i) + the float64 slack.  An empty R_i leaves the row as prepared: S_i (or +inf), cnt 0.

    Well formed.  The first min(cnt, cap) entries have a non-zero mask whose columns col + b lie in R_i, and no
    column is admitted twice: every (row, column) pair is scanned by exactly one item (times == 1), and one scan
    emits a chunk at most once, so a duplicate means an item (or a tile) ran twice.

    Complete (cnt <= cap).  Every j in R_i with a_ij + g_i <= threshold_lo(row_min_i) is admitted.  Every mask is
    built against, and every staged chunk is kept or dropped against, nn_threshold(s) for an s the CTA holds at that
    moment: the seed, a value max(v + nx, 0) of its own scan, or a value it read from row_min_bits.  Each of these is
    >= the final shared minimum, which is the atomicMin over all of them, and nn_threshold is monotone in s, so every
    threshold applied is >= nn_threshold(row_min) >= threshold_lo(row_min).  The column's fp32 value is <= a_ij + g_i
    <= that bound: its chunk's minimum is inside every threshold the chunk meets, the chunk survives staging and
    compaction, and its bit is set.

    Sound.  Every admitted j has a_ij - g_i <= threshold_hi(max(m_c + g_i + nx_i, 0) (1 + 2^-22)), m_c the smallest
    a over the columns of its chunk that the emitting item scanned (all bits of one entry come from one item): a chunk is recorded only once its own minimum has moved the running minimum
    (or a smaller value had), so its mask's threshold comes from an s <= max(fp32 chunk minimum + nx, 0).

    Non-vacuous.  required_extra counts the pairs completeness required beyond each row's argmin; outside counts the
    in-range columns of admitted chunks that the sound bound excludes (what an exact mask must drop)."""
    m, n = a.shape
    rep = Report()
    nx, g = win.nx.astype(np.float64), win.g.astype(np.float64)
    rmin = np.asarray(row_min_bits, dtype=np.uint32).view(np.float32)
    seed = None if seed_bits is None else np.asarray(seed_bits, dtype=np.uint32)
    cnt_all = np.asarray(cand_cnt, dtype=np.int64)
    idx = np.asarray(cand_idx, dtype=np.int32).reshape(m, cap, 2)
    if times is not None:
        for i, j in zip(*np.nonzero(times > 1)):
            rep.add("pair scanned by more than one item (the work list breaks its contract)", i, j, owner[i, j])
    for i in range(m):
        R = inr[i]
        cnt = int(cnt_all[i])
        s_bits = INF_BITS if seed is None else int(seed[i])
        if not R.any():
            if int(rmin[i:i + 1].view(np.uint32)[0]) != s_bits:
                rep.add("row_min changed on a row with an empty range", i, value=float(rmin[i]),
                        bound=float(np.uint32(s_bits).view(np.float32)))
            if cnt != 0:
                rep.add("candidates on a row with an empty range", i, value=cnt, bound=0)
            continue
        rep.checked_rows += 1
        ai = a[i]
        cols_r = np.flatnonzero(R)
        j_min = int(cols_r[np.argmin(ai[cols_r])])
        mu = float(ai[j_min])
        want = max(mu + nx[i], 0.0)
        if seed is not None:
            want = min(want, float(np.uint32(s_bits).view(np.float32)))
        bound = g[i] + 2.0 ** -22 * (abs(mu) + nx[i]) + float(slack[i, cols_r].max())
        got = float(rmin[i])
        err = abs(got - want) if np.isfinite(got) else np.inf
        rep.rowmin_frac = max(rep.rowmin_frac, err / bound if bound > 0 else (0.0 if err == 0 else np.inf))
        if not err <= bound:
            rep.add("row_min off the range's minimum", i, j_min, owner[i, j_min], got, want)
        # lists
        if cnt < 0:
            rep.add("negative candidate count", i, value=cnt)
            continue
        if cnt > cap:
            rep.overflowed += 1
        seen = np.zeros(n, dtype=bool)
        for k in range(min(cnt, cap)):
            col, mask = int(idx[i, k, 0]), int(idx[i, k, 1]) & 0xFFFFFFFF
            if mask == 0:
                rep.add("entry with an empty mask", i, col)
                continue
            bits = col + np.flatnonzero((mask >> np.arange(CHUNK, dtype=np.uint64)) & 1)
            ok = (bits >= 0) & (bits < n)
            for j in bits[~ok]:
                rep.add("bit outside the train rows", i, j)
            bits = bits[ok]
            for j in bits[~R[bits]]:
                rep.add("bit outside the row's range", i, j, owner[i, j])
            for j in bits[seen[bits]]:
                rep.add("column admitted twice", i, j, owner[i, j])
            seen[bits] = True
            # sound: against the widest window of the chunk's own minimum, over the columns the emitting item scanned
            # (a span may end mid-chunk, and the next item's columns are not part of this chunk)
            adm = bits[R[bits]]
            if adm.size == 0:
                continue
            w = np.unique(owner[i, adm])
            if w.size != 1:
                rep.add("entry mixes the columns of several items", i, col, int(w[0]))
                continue
            ch = np.arange(col, col + CHUNK)
            ch = ch[(ch >= 0) & (ch < n)]
            ch = ch[R[ch] & (owner[i, ch] == w[0])]
            s_hi = max(float(ai[ch].min()) + g[i] + nx[i], 0.0) * (1 + 2.0 ** -22)
            t_hi = threshold_hi(s_hi, nx[i], float(win.e2_hi[i]), g[i])
            over = ai[adm] - g[i] - slack[i, adm] > t_hi
            for j in adm[over]:
                rep.add("admitted column outside its chunk's window", i, j, owner[i, j], ai[j] - g[i], t_hi)
            rep.outside += int(np.sum(ai[ch] - g[i] > t_hi))
        if cnt > cap:
            continue
        t_lo = float(threshold_lo(F32(got), win.nx[i], win.e2_lo[i], win.g[i])) if np.isfinite(got) else np.inf
        need = R & (ai + g[i] + slack[i] <= t_lo)
        for j in np.flatnonzero(need & ~seen):
            rep.add("required column missing from the list", i, j, owner[i, j], ai[j] + g[i], t_lo)
        rep.required_extra += int(need.sum()) - int(need[j_min])
    return rep
