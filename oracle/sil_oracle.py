"""float64 references of the silhouette pass (tip_sil_prep -> tip_sil_dsum -> tip_sil_finish) (TEST INFRASTRUCTURE ONLY).

Written from sklearn's `silhouette_samples` and from the operand layout that include/b200tip.h and DESIGN.md §2 / §4b
document, not from the CUDA:

  * `pack_sil`       the three-segment split-bf16 operands of `tip_sil_prep`, emulated in NumPy;
  * `exact_dsum`     per-(slot, row) sums over a work item's column span of exact Euclidean distances, own column excluded;
  * `silhouette_from_sums` / `exact_silhouette`   sklearn's silhouette from per-cluster distance sums / from the input;
  * `finish_replica` `tip_sil_finish`'s double arithmetic restated in NumPy, in the documented order, to compare bit for bit.

Error budget of the exact case (`dsum_bound`).  With integer rows |x| <= 8 plus a shift of 64 on one coordinate of the
column role (|y| <= 72), every bf16 operand is exact (integers up to 256 are), the low parts l are 0, and every product,
partial sum and norm of the K-loop is an integer below 2^24 in magnitude for d <= 2048: the fp32 accumulator, the
norm add and the clamp are exact in any order, so the squared distance reaching the epilogue is exact.  What remains:
  * sqrt.approx.f32 is an approximation with a bounded relative error, not a correctly rounded sqrt (PTX ISA); the
    budget takes 4 ulp, 4 * 2^-23 = 4.8e-7 relative, twice the 2 ulp the kernel's own comment assumes;
  * the 32-column chunk sum in fp32 (eight values per lane in a depth-3 tree, then two quad shuffles): a tree of
    depth 5 over non-negative terms, at most 5 * 2^-24 = 3.0e-7 relative;
  * the chunk sums are added in double (relative error below 2^-40 for any span) and the span's sum is cast to
    float once: 2^-24 = 6.0e-8 relative.
Together about 8.4e-7 of the exact sum; `dsum_bound` uses beta = 1e-6.

Inputs are NumPy arrays (the distance sums also take a torch device to run on); nothing in the product package
imports this module.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

BETA = 1e-6        # relative error budget of one exact-case (slot, row) distance sum, derived above
INT_RANGE = 8      # exact-case rows: integers in [-INT_RANGE, INT_RANGE]
INT_SHIFT = 64     # column role: y_i = x_i + INT_SHIFT * e_(i mod d)


# ---- operand packing -------------------------------------------------------------------------------------------
def pair_pitch(d: int) -> int:
    """row pitch of the three-segment operand in elements: 3 * d16 + a 16-wide tail, rounded up to 64"""
    d16 = -(-d // 16) * 16
    return (3 * d16 + 16 + 63) // 64 * 64


def bf16_rn(v: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 by round to nearest even, returned as float32 values (finite inputs)"""
    u = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32)
    r = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return r.view(np.float32)


def bf16_bits(v: np.ndarray) -> np.ndarray:
    """the bfloat16 bit patterns of float32 values that are bf16-exact"""
    u = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32)
    assert not np.any(u & np.uint32(0xFFFF)), "value is not bf16-exact"
    return (u >> np.uint32(16)).astype(np.uint16)


def split3(t: np.ndarray) -> np.ndarray:
    """3-way bf16 split of fp32 values: c0 = bf16(t), c1 = bf16(t - c0), c2 = bf16((t - c0) - c1), all in fp32"""
    t = np.asarray(t, dtype=np.float32)
    c0 = bf16_rn(t)
    r = t - c0
    c1 = bf16_rn(r)
    c2 = bf16_rn(r - c1)
    return np.stack([c0, c1, c2], axis=-1)


def pack_sil(x: np.ndarray, center: Optional[np.ndarray] = None,
             order: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """NumPy emulation of tip_sil_prep on rows x[order] (float32 / float64, [n, d]); center: d float32 values or None.
    Returns (q_pack, t_pack) as uint16 bf16 bit patterns [n, pitch] and sqnorm (float32 [n]):
      v = fl32(x - c) (float32: one fp32 subtraction; float64: the double difference rounded once),
      h = bf16(v), l = bf16(v - h), padded with zeros from d to d16 = round_up(d, 16);
      query row [h | l | h | 1, 1, 1, 0...], train row [-2h | -2h | -2l | split3(T) | 0...],
      T = sum(h^2 + 2 h l) in double, rounded to fp32 (the norm the operands carry: identical rows cancel)."""
    x = np.asarray(x)
    assert x.dtype in (np.float32, np.float64) and x.ndim == 2
    if order is not None:
        x = x[np.asarray(order)]
    n, d = x.shape
    d16 = -(-d // 16) * 16
    pitch = pair_pitch(d)
    c = np.zeros(d, dtype=np.float32) if center is None else np.asarray(center, dtype=np.float32)
    if x.dtype == np.float32:
        v = x - c
    else:
        v = (x - c.astype(np.float64)).astype(np.float32)
    vp = np.zeros((n, d16), dtype=np.float32)
    vp[:, :d] = v
    h = bf16_rn(vp)
    lo = bf16_rn(vp - h)                  # v - h is exact in fp32
    hd, ld = h.astype(np.float64), lo.astype(np.float64)
    t = np.sum(hd * hd + 2.0 * hd * ld, axis=1).astype(np.float32)
    q = np.zeros((n, pitch), dtype=np.float32)
    q[:, :d16], q[:, d16:2 * d16], q[:, 2 * d16:3 * d16] = h, lo, h
    q[:, 3 * d16:3 * d16 + 3] = 1.0
    m2 = np.float32(-2.0)
    tr = np.zeros((n, pitch), dtype=np.float32)
    tr[:, :d16], tr[:, d16:2 * d16], tr[:, 2 * d16:3 * d16] = m2 * h, m2 * h, m2 * lo
    tr[:, 3 * d16:3 * d16 + 3] = split3(t)
    return bf16_bits(q), bf16_bits(tr), t


# ---- exact distances and sums ----------------------------------------------------------------------------------
def _torch64(a, device):
    import torch

    return torch.as_tensor(np.asarray(a, dtype=np.float64), device=device)


def _dist(a, b):
    """float64 Euclidean distances between the rows of a and b (torch): |a|^2 + |b|^2 - 2<a, b>, clamped at 0.  Exact
    (then correctly rounded by the sqrt) for integer rows; on real-valued rows the cancellation error is about
    1e-16 (|a|^2 + |b|^2) in the squared distance, so callers centre their data first."""
    import torch

    sq = (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * (a @ b.T)
    return torch.sqrt(torch.clamp_min(sq, 0.0))


def exact_dsum(xq, xt, items: np.ndarray, slots: int, device=None) -> np.ndarray:
    """float64 part[slot, row] = sum over the item's columns j in [col0, col1), j != row, of |xq_row - xt_j|, for
    every work item (tip_work_item rows: q_row0, q_rows, col0, col1, slot, flags) and every row of its tile; NaN
    where no item writes.  Queries and columns are separate matrices (rows in label-sorted order); row i's own
    column is column i."""
    n = np.asarray(xq).shape[0]
    out = np.full((slots, n), np.nan)
    spans = {}
    for q0, qr, c0, c1, slot, _ in np.asarray(items).tolist():
        rows = spans.setdefault((c0, c1, slot), np.zeros(n, dtype=bool))
        rows[q0:q0 + qr] = True
    if not spans:
        return out
    import torch

    q, t = _torch64(xq, device), _torch64(xt, device)
    idx = lambda a: torch.as_tensor(a, dtype=torch.int64, device=q.device)
    for (c0, c1, slot), mask in spans.items():
        rows = np.flatnonzero(mask)
        block = max(1, (1 << 24) // max(1, c1 - c0))
        for b0 in range(0, rows.size, block):
            r = rows[b0:b0 + block]
            dist = _dist(q[idx(r)], t[c0:c1])
            own = np.flatnonzero((r >= c0) & (r < c1))
            dist[idx(own), idx(r[own] - c0)] = 0.0
            out[slot, r] = dist.sum(1).cpu().numpy()
    return out


def check_work_list(items: np.ndarray, slot_cluster: np.ndarray, counts: Sequence[int], span_tiles: int,
                    row_tile: int = 128, col_tile: int = 256) -> None:
    """Asserts what the silhouette pass needs of its work list, independently of how it was built (exact_dsum follows
    whatever list it is given): slot_cluster is non-decreasing; every slot is ONE column span inside its cluster, at
    most span_tiles * col_tile wide; the spans of each non-empty cluster c tile [off[c], off[c + 1]) exactly once and no
    slot belongs to an empty cluster; every slot's query tiles (at most row_tile rows) cover rows [0, n) exactly once."""
    items = np.asarray(items, dtype=np.int64)
    slot_cluster = np.asarray(slot_cluster)
    counts = np.asarray(counts, dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(counts)])
    n = int(off[-1])
    slots = slot_cluster.shape[0]
    assert np.all(np.diff(slot_cluster) >= 0), "slot_cluster must be non-decreasing"
    assert items.ndim == 2 and items.shape[1] == 6 and np.all((items[:, 4] >= 0) & (items[:, 4] < slots))
    span = {}
    for s in range(slots):
        sp = {(int(c0), int(c1)) for c0, c1 in items[items[:, 4] == s, 2:4]}
        assert len(sp) == 1, f"slot {s} has spans {sorted(sp)}"
        span[s] = sp.pop()
    for c in range(counts.shape[0]):
        mine = sorted(span[s] for s in np.flatnonzero(slot_cluster == c))
        if counts[c] == 0:
            assert not mine, f"empty cluster {c} has slots"
            continue
        edges = [int(off[c])] + [c1 for _, c1 in mine]
        assert [c0 for c0, _ in mine] == edges[:-1] and edges[-1] == off[c + 1], f"cluster {c}: spans {mine}"
        assert all(0 < c1 - c0 <= span_tiles * col_tile for c0, c1 in mine), f"cluster {c}: spans {mine}"
    assert np.all((items[:, 1] >= 1) & (items[:, 1] <= row_tile))
    assert np.all((items[:, 0] >= 0) & (items[:, 0] + items[:, 1] <= n))
    for s in range(slots):
        cover = np.zeros(n + 1, dtype=np.int64)
        for q0, qr in items[items[:, 4] == s, :2]:
            cover[q0] += 1
            cover[q0 + qr] -= 1
        assert np.all(np.cumsum(cover)[:n] == 1), f"slot {s}: query rows not covered exactly once"


def dsum_bound(ref: np.ndarray) -> np.ndarray:
    """per-(slot, row) error budget of a device distance sum in the exact (integer) case: BETA * ref"""
    return BETA * np.asarray(ref)


def dsum_excess(part: np.ndarray, ref: np.ndarray) -> float:
    """largest |part - ref| / dsum_bound(ref) over the written entries (inf for a non-finite part or a non-zero part
    where ref is 0); <= 1 means the device sums are inside the budget"""
    part = np.asarray(part, dtype=np.float64)
    written = ~np.isnan(ref)
    if not np.all(np.isfinite(part[written])):
        return np.inf
    err = np.abs(part[written] - ref[written])
    bound = dsum_bound(ref[written])
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    return float(ratio.max(initial=0.0))


def int_operands(counts: Sequence[int], d: int, seed: int, distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """Integer rows of the exact case, in label-sorted order: X in [-8, 8]^d, Y = X + 64 e_(i mod d).  Every own
    column |x_i - y_i| is 64 and every other |x_i - y_j| is at least 64 - 16 = 48.  distinct (d = 1): X is a set of
    distinct values (at most 17 rows), so that masking column i +- 1 instead of i changes every sum it touches."""
    rng = np.random.default_rng(seed)
    n = int(np.sum(counts))
    if distinct:
        assert d == 1 and n <= 2 * INT_RANGE + 1
        x = rng.permutation(np.arange(-INT_RANGE, INT_RANGE + 1))[:n].reshape(n, 1).astype(np.float64)
    else:
        x = rng.integers(-INT_RANGE, INT_RANGE + 1, size=(n, d)).astype(np.float64)
    y = x.copy()
    y[np.arange(n), np.arange(n) % d] += INT_SHIFT
    return x, y


def exact_layouts():
    """The layout matrix of the exact-case tests: (name, cluster sizes in label-sorted order, d, distinct rows).
    Cluster sizes on both sides of the 32-column chunk, the 128-row tile and the 256-column span unit; 64 clusters
    of mixed sizes with singletons; 500 clusters of 1-8 rows; n = 129, 4097 and 20 000; d = 1, 16 and 96 run the
    resident-query kernel, d = 97, 300 and 2048 the streaming one."""
    rng = np.random.default_rng(20261015)
    sizes = [int(s) for s in rng.permutation([1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513,
                                              4095, 4097])]
    c64 = rng.integers(2, 120, size=64)
    c64[::7] = 1
    c500 = rng.integers(1, 9, size=500)
    return [
        ("sizes_d16", sizes, 16, False),
        ("sizes_d300", sizes, 300, False),
        ("c64_d96", [int(c) for c in c64], 96, False),
        ("c64_d2048", [int(c) for c in c64], 2048, False),
        ("c500_d97", [int(c) for c in c500], 97, False),
        ("n129_128_1_d16", [128, 1], 16, False),
        ("n129_1_128_d2048", [1, 128], 2048, False),
        ("n4097_d2048", [2049, 2048], 2048, False),
        ("n4097_d96", [4096, 1], 96, False),
        ("n20000_d97", [12000, 8000], 97, False),
        ("d1_distinct", [1, 2, 5, 9], 1, True),
    ]


def layout_operands(layout) -> Tuple[np.ndarray, np.ndarray]:
    """the integer operands (X, Y) of one exact_layouts() entry: the same data on every machine"""
    _, counts, d, distinct = layout
    return int_operands(counts, d, seed=int(np.sum(counts)) * 7 + d, distinct=distinct)


# ---- silhouette ------------------------------------------------------------------------------------------------
def cluster_sums(part: np.ndarray, slot_cluster: np.ndarray, n_clusters: int) -> np.ndarray:
    """per-row distance sums per cluster [n, n_clusters] from per-slot sums [slots, n] (float64)"""
    out = np.zeros((np.asarray(part).shape[1], n_clusters))
    for s, c in enumerate(np.asarray(slot_cluster).tolist()):
        out[:, c] += np.asarray(part[s], dtype=np.float64)
    return out


def silhouette_from_sums(sums: np.ndarray, labels: np.ndarray, counts: np.ndarray) -> np.ndarray:
    """sklearn's silhouette_samples from per-row, per-cluster distance sums (own distance 0 included or not, it is 0):
    a = own sum / (n_own - 1), b = min over the other clusters of sum / n_c, (b - a) / max(a, b), NaN -> 0 (singleton
    clusters, a = b = 0).  Every cluster must be non-empty."""
    sums = np.array(sums, dtype=np.float64)
    labels = np.asarray(labels)
    counts = np.asarray(counts, dtype=np.float64)
    rows = np.arange(labels.shape[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        a = sums[rows, labels] / (counts[labels] - 1)
        sums[rows, labels] = np.inf
        b = (sums / counts).min(axis=1)
        s = (b - a) / np.maximum(a, b)
    return np.nan_to_num(s)


def exact_silhouette(x, labels, device=None, block: int = 2048) -> np.ndarray:
    """float64 silhouette_samples of the input itself (any label values), in row blocks with torch float64 on
    `device` (default: CPU).  Rows are first shifted by their mean rounded to integers (distances do not change)."""
    import torch

    lab = np.asarray(labels).reshape(-1)
    _, codes = np.unique(lab, return_inverse=True)
    counts = np.bincount(codes)
    xt = _torch64(x, device)
    xt = xt.reshape(xt.shape[0], -1)
    xt = xt - torch.round(xt.mean(dim=0))     # an integer shift: exact for integer rows and for rows near the mean
    n = xt.shape[0]
    code_t = torch.as_tensor(codes, device=xt.device)
    sums = torch.zeros((n, counts.shape[0]), dtype=torch.float64, device=xt.device)
    for r0 in range(0, n, block):
        r1 = min(n, r0 + block)
        dist = _dist(xt[r0:r1], xt)
        dist[torch.arange(r1 - r0, device=xt.device), torch.arange(r0, r1, device=xt.device)] = 0.0
        sums[r0:r1].index_add_(1, code_t, dist)
    return silhouette_from_sums(sums.cpu().numpy(), codes, counts)


def silhouette_error_bound(x, labels, device=None, block: int = 2048) -> Tuple[np.ndarray, np.ndarray]:
    """(bound, support) per row.  bound: a worst-case bound on |device silhouette - exact silhouette| from DESIGN.md
    §4b's error model, for rows that get no averaging (small clusters, d = 1).  support: the fewest rows that a or a
    possible b of the row averages over (the own cluster and every cluster that can be the nearest one within its
    error bound); rows with a large support are in the averaging regime of the §4b tolerances.
    With v = x - mean (the engine's centring) and K = 3 * d16 + 16 packed products,
    the squared distance the pass forms is off by at most E_ij = (2^-18 + (K + 16) * 2^-23) * (|v_i| + |v_j|)^2 (the
    dropped |l_i - l_j|^2, and fp32 accumulation with nothing better than truncating adds), so the distance by at most
    min(sqrt(E_ij), E_ij / d_ij) + 1e-6 * d_ij (sqrt.approx, fp32 sums).  Per row that bounds a and b by the cluster
    means da, db of those, and s = (b - a) / max(a, b) by 2 (da + db) / (max(a, b) - max(da, db)) (2 if that is not
    positive)."""
    import torch

    lab = np.asarray(labels).reshape(-1)
    _, codes = np.unique(lab, return_inverse=True)
    counts = np.bincount(codes)
    xt = _torch64(x, device)
    xt = xt.reshape(xt.shape[0], -1)
    xt = xt - xt.mean(dim=0)
    n, d = xt.shape
    gamma = 2.0 ** -18 + (3 * (-(-d // 16) * 16) + 32) * 2.0 ** -23
    norm = torch.sqrt((xt * xt).sum(1))
    code_t = torch.as_tensor(codes, device=xt.device)
    sums = torch.zeros((n, counts.shape[0]), dtype=torch.float64, device=xt.device)
    errs = torch.zeros_like(sums)
    for r0 in range(0, n, block):
        r1 = min(n, r0 + block)
        dist = _dist(xt[r0:r1], xt)
        e = gamma * (norm[r0:r1, None] + norm[None, :]) ** 2
        dd = torch.minimum(torch.sqrt(e), e / dist) + 1e-6 * dist
        diag = (torch.arange(r1 - r0, device=xt.device), torch.arange(r0, r1, device=xt.device))
        dist[diag], dd[diag] = 0.0, 0.0
        sums[r0:r1].index_add_(1, code_t, dist)
        errs[r0:r1].index_add_(1, code_t, dd)
    sums, errs = sums.cpu().numpy(), errs.cpu().numpy()
    rows = np.arange(n)
    cnt = counts.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        a, da = sums[rows, codes] / (cnt[codes] - 1), errs[rows, codes] / (cnt[codes] - 1)
        sums[rows, codes] = np.inf
        mean = sums / cnt
        pick = np.argmin(mean, axis=1)
        b = mean[rows, pick]
        emean = np.where(np.isinf(mean), 0.0, errs / cnt)
        db = np.max(emean, axis=1)                                       # any cluster may become the nearest
        m = np.maximum(a, b) - np.maximum(da, db)
        bound = np.where(m > 0, 2 * (da + db) / m, 2.0)
        # clusters that can be the nearest one within their error: mean_c - e_c <= b + e_b
        cand = mean - emean <= (b + emean[rows, pick])[:, None]
    support = np.minimum(cnt[codes], np.where(cand, cnt, np.inf).min(axis=1))
    return np.where(cnt[codes] > 1, bound, 0.0), support


def finish_replica(part: np.ndarray, slot_cluster: np.ndarray, labels_sorted: np.ndarray, counts: np.ndarray,
                   out_idx: Optional[np.ndarray]) -> np.ndarray:
    """tip_sil_finish's arithmetic in NumPy float64, in the order include/b200tip.h documents: per row, the slots of
    each cluster summed as (double) part in ascending slot order; own cluster L: a = acc / (n_L - 1) (0 if n_L <= 1);
    every other cluster c with n_c > 0: b = fmin(b, acc / n_c), starting from +inf; value (b - a) / max(a, b) when
    n_L > 1, max(a, b) > 0 and b < inf, else 0; written to out[out_idx[i]] (out_idx None: i)."""
    part = np.asarray(part, dtype=np.float32)
    slot_cluster = np.asarray(slot_cluster)
    lab = np.asarray(labels_sorted)
    counts = np.asarray(counts)
    slots, n = part.shape
    a = np.zeros(n)
    b = np.full(n, np.inf)
    acc = np.zeros(n)
    cur = int(slot_cluster[0]) if slots > 0 else -1
    for s in range(slots + 1):
        c = int(slot_cluster[s]) if s < slots else -1
        if c != cur:
            own = lab == cur
            a[own] = acc[own] / float(counts[cur] - 1) if counts[cur] > 1 else 0.0
            if counts[cur] > 0:
                b[~own] = np.fmin(b[~own], acc[~own] / float(counts[cur]))
            acc = np.zeros(n)
            cur = c
        if s < slots:
            acc = acc + part[s].astype(np.float64)
    mx = np.fmax(a, b)
    ok = (counts[lab] > 1) & (mx > 0.0) & (b < np.inf)
    v = np.zeros(n)
    with np.errstate(invalid="ignore"):
        v[ok] = (b[ok] - a[ok]) / mx[ok]
    out = np.empty(n)
    out[np.arange(n) if out_idx is None else np.asarray(out_idx)] = v
    return out
