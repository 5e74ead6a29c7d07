"""Device-side orchestration of the scoring kernels (PyTorch = memory, streams, NCCL plumbing).

Two engines sit under the reference-compatible classes in `simple_tip_b200.core`:

* `NnEngine`  — class-grouped training traces resident in HBM (original dtype for the exact
  re-rank + packed bf16 operand for the tensor-core filter); `search()` runs
  filter -> re-rank for a batch of class-sorted queries.  Used twice per DSA call
  (surprise.py:615-631: same-class nearest neighbour, then other-class nearest neighbour
  of the winning TRAIN row).
* `KdeEngine` — whitened training traces as a 3-segment split-bf16 operand; `log_kernel_sum()`
  returns per-query (max, sum) of exp(-|p_i - q_j|^2 / 2) in the log domain
  (scipy 1.4.1 gaussian_kernel_estimate, called from stable_kde.py:101).

The pure-host planning helpers (`class_layout`, `build_items`, `shard_rows`) and the
cross-rank reduction protocol (`TrainShardComm`) contain no CUDA calls and are unit-tested on
CPU (gloo, world_size 2).
"""
from __future__ import annotations

import ctypes as C
import gc
import math
import os
import re
import time
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

POOL_FRAC = 0.2           # share of the filter's work handed out dynamically
POOL_MIN_TILES = 32       # tiles per CTA below which work lists stay purely static
POOL_TILES = 4            # train tiles per dynamic item
LIVE_ITEM_TILES = 16      # train tiles per item of a live-bounded filter (DSA's stage 2 on distinct winners)
DEFAULT_CAP = 64          # candidate chunks per query (short traces)
DEFAULT_CAP_LONG = 256    # long traces: distances concentrate, more rows fall inside the window

# bench.py sets this to a list to collect (kernel name, algorithmic flops, start event, end event)
# around the tensor-core launches; None (default) records nothing.
PROFILE = None


# ------------------------------------------------------------------------------------------
# plumbing
# ------------------------------------------------------------------------------------------
def require_cuda() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("simple_tip_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _p(t: Optional[torch.Tensor]):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def tip_dtype(dt) -> int:
    if dt in (torch.float32, np.float32, np.dtype("float32")):
        return _lib.TIP_F32
    if dt in (torch.float64, np.float64, np.dtype("float64")):
        return _lib.TIP_F64
    raise TypeError(f"activation traces must be float32 or float64, got {dt}")


def to_device(a, dev: torch.device) -> torch.Tensor:
    """Host -> HBM.  Pinned sources (e.g. views of torch pinned tensors) copy asynchronously.
    Traces that already live on the GPU (torch CUDA tensors) are used in place."""
    if isinstance(a, torch.Tensor):
        return a.to(dev, non_blocking=True).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)


def device_matrix(layers) -> Optional[torch.Tensor]:
    """Activation traces handed over as device tensors (one [N, ...] tensor or a list of them, the
    form a forward hook produces): the flattened [N, D] matrix on the GPU, else None.  Mirrors
    `_flatten_layers` (surprise.py:62-66) without leaving HBM."""
    def rows(t):            # explicit width: a -1 cannot be resolved for 0 samples
        return t.reshape(t.shape[0], int(np.prod(t.shape[1:])))

    if isinstance(layers, torch.Tensor):
        return rows(layers) if layers.is_cuda else None
    if isinstance(layers, (list, tuple)) and len(layers) > 0 and all(isinstance(l, torch.Tensor) and l.is_cuda
                                                                     for l in layers):
        flat = [rows(l) for l in layers]
        return flat[0] if len(flat) == 1 else torch.cat(flat, dim=1)
    return None


def host_array(x) -> np.ndarray:
    """Labels / predictions as a NumPy array whatever they came as (device tensors are copied)."""
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return x


NP_DTYPE = {torch.float32: np.dtype(np.float32), torch.float64: np.dtype(np.float64),
            torch.float16: np.dtype(np.float16), torch.bfloat16: None}

GRAPHS = os.environ.get("B200TIP_GRAPHS", "1") != "0"   # CUDA-graph replay of repeated batch shapes


class BoundedCache(dict):
    """A dict of at most `capacity` entries: a new key that would exceed it drops the oldest entry first."""

    def __init__(self, capacity: int):
        super().__init__()
        self.capacity = capacity

    def get_or_make(self, key, make):
        if key not in self:
            if len(self) >= self.capacity:
                del self[next(iter(self))]
            self[key] = make()
        return self[key]

    def touch(self, key) -> bool:
        """True if `key` was seen before; records it either way (the seen-shape sets)."""
        seen = key in self
        self.get_or_make(key, lambda: None)
        return seen


_capture_keep: Optional[list] = None     # while capture_graphs captures: the tensors its graphs must keep alive


def keep_for_capture(*tensors) -> None:
    """Called by code that hands out a cached or engine-owned tensor.  While a CUDA graph is captured, the plan keeps
    the tensor alive, since the graph bakes in its address and a cache may evict it later.  Otherwise a no-op."""
    if _capture_keep is not None:
        _capture_keep.extend(t for t in tensors if t is not None)


def capture_graphs(segments, dev: torch.device) -> Tuple[list, list, list]:
    """segments: [(fn, capturable)].  Every fn runs once eagerly on a side stream (fills caches, sets kernel
    attributes, runs the collectives once); then each capturable fn is captured as a CUDA graph and every other fn
    runs eagerly again, which keeps the ranks' collective sequences aligned.  Returns (steps: one callable per
    segment, the graphs, the tensors keep_for_capture collected)."""
    global _capture_keep
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for fn, _ in segments:
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    steps, graphs, keep = [], [], []
    # garbage from earlier plans (graphs, their private pools) must not be released in the middle of a capture:
    # a cudaFree or a graph destroy there invalidates it
    gc.collect()
    was_enabled = gc.isenabled()
    gc.disable()
    try:
        for fn, capturable in segments:
            if not capturable:
                fn()
                steps.append(fn)
                continue
            g = torch.cuda.CUDAGraph()
            _capture_keep = keep
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                fn()
            _capture_keep = None
            steps.append(g.replay)
            graphs.append(g)
    finally:
        _capture_keep = None
        if was_enabled:
            gc.enable()
    return steps, graphs, keep


# ------------------------------------------------------------------------------------------
# host-side planning (no CUDA)
# ------------------------------------------------------------------------------------------
def class_layout(labels: np.ndarray, num_classes: int) -> Tuple[np.ndarray, np.ndarray]:
    """Stable grouping by class.  Returns (order, offsets[num_classes+1]); `order` lists the
    positions of rows with 0 <= label < num_classes, grouped by class, ascending position inside
    a class (the order `np.argwhere(pred == label)` gives, surprise.py:554,581)."""
    labels = np.asarray(labels)
    ok = (labels >= 0) & (labels < num_classes)
    # NumPy's stable sort is a radix sort for <= 16-bit integers: ~10x faster than on int64
    small = np.uint16 if num_classes <= 65535 else np.int64
    if ok.all():
        keys = labels.astype(small)
        order = np.argsort(keys, kind="stable")
        counts = np.bincount(keys, minlength=num_classes)[:num_classes]
    else:
        valid = np.flatnonzero(ok)
        keys = labels[valid].astype(small)
        order = valid[np.argsort(keys, kind="stable")]
        counts = np.bincount(keys, minlength=num_classes)[:num_classes]
    offsets = np.zeros(num_classes + 1, dtype=np.int64)
    np.cumsum(counts, out=offsets[1:])
    return order, offsets


def shard_rows(labels: np.ndarray, num_classes: int, rank: int, world: int) -> np.ndarray:
    """Rows of the training set kept by `rank`: every class is dealt round-robin, so each rank
    holds ~N_c/world rows of every class in ascending original order."""
    order, off = class_layout(labels, num_classes)
    keep = []
    for c in range(num_classes):
        rows = order[off[c]:off[c + 1]]
        keep.append(rows[rank::world])
    return np.sort(np.concatenate(keep)) if keep else np.zeros(0, dtype=np.int64)


def span_tiles_for(total_tile_pairs: int, sms: int, per_sm: int = 6, lo: int = 2, hi: int = 16) -> int:
    """Column tiles per work item: aim for ~per_sm items per SM so the static round-robin balances."""
    return int(min(hi, max(lo, round(total_tile_pairs / max(1, sms * per_sm)))))


def build_items(q_off: np.ndarray, ranges_per_class: Sequence[Sequence[Tuple[int, int]]], span_tiles: int,
                row_tile: int = _lib.ROW_TILE, col_tile: int = _lib.COL_TILE) -> Tuple[np.ndarray, int]:
    """Work list of the tensor-core pass.  q_off[c]..q_off[c+1] are the (class-sorted) query rows
    of class c; ranges_per_class[c] the train-row ranges they must be compared with.  Every item is
    one row_tile-row query tile x one span of at most span_tiles*col_tile train rows.  Returns
    (int32 array [n, 6] laid out as tip_work_item, max number of spans per class)."""
    width = span_tiles * col_tile
    out = []
    max_slots = 1
    for c, ranges in enumerate(ranges_per_class):
        cnt = int(q_off[c + 1] - q_off[c])
        if cnt <= 0:
            continue
        spans = []
        for lo, hi in ranges:
            for s in range(int(lo), int(hi), width):
                spans.append((s, min(s + width, int(hi))))
        if not spans:
            continue
        max_slots = max(max_slots, len(spans))
        r0 = np.arange(int(q_off[c]), int(q_off[c + 1]), row_tile, dtype=np.int64)
        rows = np.minimum(row_tile, int(q_off[c + 1]) - r0)
        sp = np.asarray(spans, dtype=np.int64)
        nt, ns = r0.shape[0], sp.shape[0]
        item = np.zeros((nt * ns, 6), dtype=np.int32)
        item[:, 0] = np.repeat(r0, ns)
        item[:, 1] = np.repeat(rows, ns)
        item[:, 2] = np.tile(sp[:, 0], nt)
        item[:, 3] = np.tile(sp[:, 1], nt)
        item[:, 4] = np.tile(np.arange(ns), nt)
        out.append(item)
    if not out:
        return np.zeros((0, 6), dtype=np.int32), max_slots
    return np.concatenate(out), max_slots


def build_other_class_items(q_off: np.ndarray, t_off: np.ndarray, row_tile: int, col_tile: int, span_of) -> np.ndarray:
    """Work list of DSA's second stage (every query against the train rows of all OTHER classes,
    surprise.py:622-629).  Queries are tiled in class-sorted order regardless of class boundaries, so
    tiles are full however many classes there are.  A tile whose queries share one class scans the
    two train ranges around that class; a tile that mixes classes scans every train row and each
    query masks out its own class in the epilogue (item flag bit 0)."""
    q_off = np.asarray(q_off, dtype=np.int64)
    t_off = np.asarray(t_off, dtype=np.int64)
    m, n = int(q_off[-1]), int(t_off[-1])
    if m == 0 or n == 0:
        return np.zeros((0, 6), dtype=np.int32)
    starts = np.arange(0, m, row_tile, dtype=np.int64)
    rows = np.minimum(row_tile, m - starts)
    first_cls = np.searchsorted(q_off, starts, side="right") - 1
    last_cls = np.searchsorted(q_off, starts + rows - 1, side="right") - 1
    single = first_cls == last_cls
    cols = np.where(single, n - (t_off[np.minimum(first_cls + 1, len(t_off) - 1)] - t_off[first_cls]), n)
    pairs = int(np.sum(np.ceil(cols / col_tile)))
    width = span_of(pairs) * col_tile
    out = []
    for r0, nr, c, one in zip(starts, rows, first_cls, single):
        ranges = [(0, int(t_off[c])), (int(t_off[c + 1]), n)] if one else [(0, n)]
        spans = [(s0, min(s0 + width, hi)) for lo, hi in ranges for s0 in range(lo, hi, width)]
        if not spans:
            continue
        item = np.zeros((len(spans), 6), dtype=np.int32)
        item[:, 0], item[:, 1] = r0, nr
        item[:, 2:4] = np.asarray(spans, dtype=np.int64)
        item[:, 4] = np.arange(len(spans))
        item[:, 5] = 0 if one else 1
        out.append(item)
    return np.concatenate(out) if out else np.zeros((0, 6), dtype=np.int32)


def query_tiles(q_off: np.ndarray, ranges_per_class, t_off: Optional[np.ndarray], row_tile: int, mixed: bool):
    """Query tiles of one search stage as (first row, rows, train ranges, flag) tuples.
    mixed=False: class-aligned tiles (a tile never crosses a class boundary) scanning the ranges of
    their class.  mixed=True (DSA's other-class stage with few queries per class): tiles cut
    regardless of class boundaries; a tile that mixes classes scans every train row and each query
    masks its own class in the epilogue (flag bit 0)."""
    q_off = np.asarray(q_off, dtype=np.int64)
    tiles = []
    if not mixed:
        for c, ranges in enumerate(ranges_per_class):
            rs = [(int(lo), int(hi)) for lo, hi in ranges if int(hi) > int(lo)]
            if not rs:
                continue
            for r0 in range(int(q_off[c]), int(q_off[c + 1]), row_tile):
                tiles.append((r0, min(row_tile, int(q_off[c + 1]) - r0), rs, 0))
        return tiles
    t_off = np.asarray(t_off, dtype=np.int64)
    m, n = int(q_off[-1]), int(t_off[-1])
    for r0 in range(0, m, row_tile):
        nr = min(row_tile, m - r0)
        c0 = int(np.searchsorted(q_off, r0, side="right") - 1)
        c1 = int(np.searchsorted(q_off, r0 + nr - 1, side="right") - 1)
        if c0 == c1:
            rs = [(lo, hi) for lo, hi in ((0, int(t_off[c0])), (int(t_off[c0 + 1]), n)) if hi > lo]
            flag = 0
        else:
            rs, flag = ([(0, n)] if n > 0 else []), 1
        if rs:
            tiles.append((r0, nr, rs, flag))
    return tiles


def build_balanced_items(tiles, col_tile: int, n_cta: int, item_cost: float = 0.75, pool_frac: float = 0.0,
                         pool_tiles: int = 4) -> Tuple[np.ndarray, int]:
    """Work list for the persistent resident-query kernel.  Returns (items [n, 6], n_static).

    Static part, balanced for the kernel's schedule (CTA b runs items b, b + G, b + 2G, ...;
    G = min(n_cta, #items)): the (query tile x train tile) pairs are linearised query-tile-major
    and cut into G contiguous chunks of equal cost, so every CTA streams the same number of train
    tiles (+-1) and loads as few query tiles as possible; a chunk becomes one item per (query tile,
    train range) it touches.  `item_cost` is the price of starting an item (query-tile load +
    pipeline refill) in train-tile units.

    Dynamic part: the last `pool_frac` of every chunk is cut off and split into items of at most
    `pool_tiles` train tiles that follow the static items in the array; CTAs pull them through an
    atomic counter when their static share is done, which absorbs run-time differences between
    CTAs (data-dependent candidate handling) that no static cut can foresee."""
    segs = []          # (q_row0, q_rows, lo, hi, flag, ntiles)
    for r0, nr, ranges, flag in tiles:
        for lo, hi in ranges:
            nt = -(-(int(hi) - int(lo)) // col_tile)
            if nt > 0:
                segs.append((int(r0), int(nr), int(lo), int(hi), int(flag), nt))
    if not segs:
        return np.zeros((0, 6), dtype=np.int32), 0
    total = sum(sg[5] for sg in segs)
    g = int(min(n_cta, total))
    # Cost axis: every segment costs item_cost up front, then 1 per train tile.  A tile belongs to
    # the CTA whose equal share of the axis holds the tile's centre; consecutive tiles of a
    # segment with the same owner form one piece.
    cost_total = total + item_cost * len(segs)
    per_cta = [[] for _ in range(g)]           # pieces: (segment index, first tile, one past last tile)
    pos = 0.0
    for si, (r0, nr, lo, hi, flag, nt) in enumerate(segs):
        pos += item_cost
        owner = np.minimum(((pos + np.arange(nt) + 0.5) * (g / cost_total)).astype(np.int64), g - 1)
        cuts = np.flatnonzero(np.diff(owner)) + 1
        starts = np.concatenate(([0], cuts))
        ends = np.concatenate((cuts, [nt]))
        for t0, t1 in zip(starts, ends):
            per_cta[int(owner[t0])].append((si, int(t0), int(t1)))
        pos += nt

    def as_item(si, t0, t1):
        r0, nr, lo, hi, flag, _ = segs[si]
        return (r0, nr, lo + t0 * col_tile, min(hi, lo + t1 * col_tile), 0, flag)

    pool, tails = [], []
    if pool_frac > 0.0 and total >= POOL_MIN_TILES * g:   # short launches: the item-start cost outweighs the tail
        for lst in per_cta:
            give = int(round(pool_frac * sum(t1 - t0 for _, t0, t1 in lst)))
            tail = []
            while give > 0 and lst:
                si, t0, t1 = lst[-1]
                take = min(give, t1 - t0)
                tail.append((si, t1 - take, t1))
                give -= take
                if take == t1 - t0:
                    lst.pop()
                else:
                    lst[-1] = (si, t0, t1 - take)
            mine = []
            for si, t0, t1 in reversed(tail):             # keep the train order inside a chunk
                for p0 in range(t0, t1, pool_tiles):
                    mine.append(as_item(si, p0, min(t1, p0 + pool_tiles)))
            tails.append(mine)
        # Pool order: round-robin over the chunks.  CTAs arrive at the pool at about the same time and
        # take one item per round, so a CTA's successive draws tend to be successive pieces of one
        # chunk's tail — same query tile, which the kernel then keeps resident.
        for r in range(max((len(tl) for tl in tails), default=0)):
            pool.extend(tl[r] for tl in tails if len(tl) > r)
    per_cta = [[as_item(*pc) for pc in lst] for lst in per_cta if lst]
    per_cta.sort(key=len, reverse=True)       # CTAs with more items first: rounds stay dense prefixes
    g = len(per_cta)
    rounds = len(per_cta[0]) if per_cta else 0
    out = []
    empty = (0, 0, 0, 0, 0, 0)                # col0 == col1: the kernel skips it
    for r in range(rounds):
        row = [lst[r] for lst in per_cta if len(lst) > r]
        if r + 1 < rounds or pool:
            row += [empty] * (g - len(row))   # keep item index = round * G + CTA
        out.extend(row)
    n_static = len(out)
    out.extend(pool)
    return np.asarray(out, dtype=np.int32).reshape(-1, 6), n_static


def build_live_items(q_off: np.ndarray, ranges_per_class, row_tile: int, col_tile: int,
                     item_tiles: int = LIVE_ITEM_TILES) -> np.ndarray:
    """Work list of a filter whose queries end at a bound only the device knows (tip_nn_filter_live: DSA's stage 2
    on the distinct stage-1 winners, which fill each class's slot range from its start).  Every item is drawn from
    the pool (n_static = 0) and covers one class-aligned query tile x at most `item_tiles` train tiles.  Items are
    ordered by the query tile's index inside its class, then class, then train row: the first tiles of every class
    are the likeliest to hold live rows, so live work comes first and the items past the bounds cluster at the end,
    where skipping them only costs CTAs that have nothing left to do."""
    q_off = np.asarray(q_off, dtype=np.int64)
    width = item_tiles * col_tile
    keyed = []
    for c, ranges in enumerate(ranges_per_class):
        spans = [(s0, min(s0 + width, int(hi))) for lo, hi in ranges for s0 in range(int(lo), int(hi), width)]
        for j, r0 in enumerate(range(int(q_off[c]), int(q_off[c + 1]), row_tile)):
            nr = min(row_tile, int(q_off[c + 1]) - r0)
            keyed.extend(((j, c, s0), (r0, nr, s0, s1, 0, 0)) for s0, s1 in spans)
    keyed.sort(key=lambda kv: kv[0])
    return np.asarray([it for _, it in keyed], dtype=np.int32).reshape(-1, 6)


def span_major(items: np.ndarray) -> np.ndarray:
    """Order the streaming kernel's work list by (train span, query tile).  CTA b runs items b, b + G, ...,
    so the CTAs that run at the same time then scan the SAME train rows for different query tiles: a train
    tile comes out of HBM once and is shared through L2.  Query-tile-major order re-reads the whole packed
    training set from HBM for every 128-row query tile — at C5's size (2.7 GB per rank) that made the
    tensor-core pass HBM-bound at 128 flop/B (measured: 42 ms instead of 26 for 10k x 640k x 2048)."""
    if items.shape[0] < 2:
        return items
    return np.ascontiguousarray(items[np.lexsort((items[:, 0], items[:, 2]))])


def count_tile_pairs(q_off: np.ndarray, ranges_per_class, row_tile: int = _lib.ROW_TILE,
                     col_tile: int = _lib.COL_TILE) -> int:
    total = 0
    for c, ranges in enumerate(ranges_per_class):
        cnt = int(q_off[c + 1] - q_off[c])
        if cnt <= 0:
            continue
        cols = sum(max(0, int(hi) - int(lo)) for lo, hi in ranges)
        total += math.ceil(cnt / row_tile) * math.ceil(cols / col_tile)
    return total


# ------------------------------------------------------------------------------------------
# cross-rank protocol (N_train sharded over the ranks of one NVSwitch box)
# ------------------------------------------------------------------------------------------
# "This shard has no row of that range" is a quiet NaN's bit pattern, which lies above +inf's: a real distance can
# be +inf (float32 traces whose squared differences overflow), and unsigned / non-negative integer order then still
# puts every real distance, +inf included, ahead of "none" (csrc/shard.cu uses the same patterns).
KEY_NONE_HI32 = 0x7FC00000
KEY_NONE_HI64 = 0x7FF8000000000000
KEY_INF_HI32 = 0x7F800000
KEY_INF_HI64 = 0x7FF0000000000000
KEY_NONE_LO = 0x7FFFFFFF
P2P_MIN_RECORDS = 1 << 18            # receive slots per rank: 2 x world x 4 MiB


def dist_keys(dist: torch.Tensor, none: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Non-negative float32 / float64 distances as int32 / int64 bit patterns that order like the distances, NaN
    (and rows flagged in `none`) replaced by the "no row" pattern above +inf.  An integer MIN over shards of these
    keys is the minimum distance, with +inf kept and "none" only where no shard had a row."""
    f32 = dist.dtype == torch.float32
    assert f32 or dist.dtype == torch.float64
    bits = dist.contiguous().view(torch.int32 if f32 else torch.int64)
    empty = torch.isnan(dist) if none is None else torch.isnan(dist) | none
    return torch.where(empty, torch.full_like(bits, KEY_NONE_HI32 if f32 else KEY_NONE_HI64), bits)


def keys_dist(keys: torch.Tensor) -> torch.Tensor:
    """Inverse of dist_keys: int32 keys -> float32, int64 -> float64, "no row" (anything above +inf) -> NaN."""
    f32 = keys.dtype == torch.int32
    assert f32 or keys.dtype == torch.int64
    keys = keys.contiguous()
    dist = keys.view(torch.float32 if f32 else torch.float64)
    return torch.where(keys > (KEY_INF_HI32 if f32 else KEY_INF_HI64), torch.full_like(dist, float("nan")), dist)


def pack_winner_keys(dist: torch.Tensor, gid: torch.Tensor) -> torch.Tensor:
    """float32 distances (>= 0, NaN = no row on this shard) and original indices -> int64 keys
    (dist_keys << 32 | index).  Non-negative IEEE floats order like their bit patterns and the
    sign bit is clear, so ONE integer MIN all-reduce yields np.min and np.argmin's first occurrence
    (surprise.py:645-647) over all shards.  Plain torch ops: runs on CPU (gloo test) and CUDA."""
    assert dist.dtype == torch.float32
    none = torch.isnan(dist) | (gid < 0)
    hi = dist_keys(dist, none).to(torch.int64)
    lo = torch.where(none, torch.full_like(gid, KEY_NONE_LO, dtype=torch.int64), gid.to(torch.int64))
    return (hi << 32) | lo


def unpack_winner_keys(keys: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Inverse of pack_winner_keys: (float32 distance with NaN for 'no row anywhere', int64 index or -1)."""
    hi = (keys >> 32).to(torch.int32)
    lo = keys & 0xFFFFFFFF
    none = (hi > KEY_INF_HI32) | (lo >= KEY_NONE_LO)
    dist = torch.where(none, torch.full((), float("nan"), dtype=torch.float32, device=keys.device), keys_dist(hi))
    return dist, torch.where(none, torch.full_like(lo, -1), lo)


WINNER_NONE = torch.iinfo(torch.int64).max


def winner_index_candidates(local: torch.Tensor, gkey: torch.Tensor, gid: torch.Tensor) -> torch.Tensor:
    """Second step of the float64 winner exchange: this rank's original index where its dist_keys `local` hold
    the global minimum `gkey` (a real row, +inf included), else WINNER_NONE; a MIN over the ranks is then
    np.argmin's first occurrence."""
    mine = (local == gkey) & (local <= KEY_INF_HI64) & (gid >= 0)
    return torch.where(mine, gid.to(torch.int64), torch.full_like(gid, WINNER_NONE, dtype=torch.int64))


def winner_from_keys(gkey: torch.Tensor, ggid: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(global minimum key, reduced winner_index_candidates) -> (float64 distance, int64 index); "none" is
    decided by the index alone: NaN / -1 where no rank had a row."""
    none = ggid == WINNER_NONE
    dist = keys_dist(gkey)
    return (torch.where(none, torch.full_like(dist, float("nan")), dist),
            torch.where(none, torch.full_like(ggid, -1), ggid))


class P2PExchange:
    """Symmetric receive buffers of libb200tip's tip_comm, one per rank, opened across the
    processes of one box with CUDA IPC; the handles travel through torch.distributed once."""

    def __init__(self, dist, group, dev: torch.device, cap_records: int):
        self.lib = _lib.load()
        self.cap = int(cap_records)
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.handle = None
        self.local = C.c_void_p(0)
        handle = (C.c_ubyte * 64)()
        rc = self.lib.tip_comm_alloc(self.world, self.cap, C.byref(self.local), handle)
        ok = torch.tensor([1 if rc == 0 else 0], dtype=torch.int32, device=dev)
        mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=dev)
        every = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(every, mine, group=group)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        err = None
        if int(ok.item()) == 1:
            blob = b"".join(bytes(t.cpu().numpy().tobytes()) for t in every)
            out = C.c_void_p(0)
            rc = self.lib.tip_comm_open(self.rank, self.world, self.local, blob, self.cap, C.byref(out))
            if rc == 0:
                self.handle = out
            else:
                err = self.lib.tip_last_error().decode(errors="replace")
        else:
            err = "tip_comm_alloc failed on some rank"
        ok = torch.tensor([1 if self.handle is not None else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)       # all ranks take the same path
        if int(ok.item()) != 1:
            self.close()
            raise RuntimeError(f"peer-memory exchange unavailable: {err or 'a peer could not map the buffers'}")

    def close(self):
        if self.handle is not None:
            self.lib.tip_comm_close(self.handle)
            self.handle = None
        if self.local:
            self.lib.tip_comm_free_local(self.local)
            self.local = C.c_void_p(0)

    def push_nn(self, dist_t: torch.Tensor, gid: Optional[torch.Tensor]):
        _lib.check(self.lib.tip_comm_push_nn(self.handle, _p(dist_t), tip_dtype(dist_t.dtype), _p(gid), dist_t.shape[0],
                                             _stream()), "tip_comm_push_nn")

    def min_into(self, out: torch.Tensor):
        _lib.check(self.lib.tip_comm_min(self.handle, tip_dtype(out.dtype), out.shape[0], _p(out), _stream()), "tip_comm_min")

    def lse(self, mx: torch.Tensor, sm: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        m = mx.shape[0]
        _lib.check(self.lib.tip_comm_push_lse(self.handle, _p(mx), _p(sm), m, _stream()), "tip_comm_push_lse")
        gm = torch.empty(m, dtype=torch.float32, device=mx.device)
        gs = torch.empty(m, dtype=torch.float64, device=mx.device)
        _lib.check(self.lib.tip_comm_lse(self.handle, m, _p(gm), _p(gs), _stream()), "tip_comm_lse")
        return gm, gs


class TrainShardComm:
    """Exchange steps of the N_train-sharded search over a torch.distributed group.

    On GPUs of one NVSwitch box the per-query records travel as peer stores fused into our own
    kernels (`P2PExchange`, csrc/shard.cu); otherwise — gloo in the CPU tests, B200TIP_EXCHANGE=nccl,
    or no peer access — as ONE integer MIN all-reduce per stage through torch.distributed.  All
    messages are O(N_test) scalars; the stage-2 query rows are gathered from the replicated raw
    training set by original index (or, without a replica, summed from their owners)."""

    def __init__(self, group=None, exchange: Optional[str] = None):
        import torch.distributed as dist

        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self.dist = dist
        self.group = group
        self.exchange = exchange or os.environ.get("B200TIP_EXCHANGE", "auto")     # auto | p2p | nccl
        assert self.exchange in ("auto", "p2p", "nccl"), self.exchange
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.collectives = 0          # torch.distributed all-reduces issued on the data path
        self._p2p = None
        self._p2p_failed = None

    # -- peer-memory exchange -----------------------------------------------------------------
    def p2p(self, dev: torch.device, records: int) -> Optional[P2PExchange]:
        """The peer-memory exchange sized for `records` queries, or None (collective fallback).
        Collective: every rank must call it with the same arguments."""
        if self.exchange == "nccl" or self.world < 2 or dev.type != "cuda" or self.world > 16:
            return None
        if self._p2p is not None:
            # never re-allocated: captured graphs hold its addresses.  Larger batches take the collective path.
            return self._p2p if self._p2p.cap >= records else None
        if self._p2p_failed is not None:
            return None
        try:
            self._p2p = P2PExchange(self.dist, self.group, dev, max(int(records), P2P_MIN_RECORDS))
        except (RuntimeError, _lib.TipError) as e:
            if self.exchange == "p2p":
                raise
            self._p2p_failed = str(e)
            return None
        return self._p2p

    def close(self):
        if self._p2p is not None:
            self._p2p.close()
            self._p2p = None

    def min_(self, t: torch.Tensor) -> torch.Tensor:
        self.collectives += 1
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN, group=self.group)
        return t

    def max_(self, t: torch.Tensor) -> torch.Tensor:
        self.collectives += 1
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
        return t

    def sum_(self, t: torch.Tensor) -> torch.Tensor:
        self.collectives += 1
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)
        return t

    # -- DSA stage 1: global (distance, lowest original index) and the winning rows -----------
    def reduce_winner_index(self, dist_a: torch.Tensor, gid: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Global minimum distance (NaN where no shard has a row of the class) and the original
        index of the winner — lowest index among exact ties, i.e. np.argmin's first occurrence.
        float32: one MIN all-reduce of packed 64-bit keys; float64: MIN of the distances, then MIN
        of the index among the ranks that hold the minimum."""
        if dist_a.dtype == torch.float32:
            return unpack_winner_keys(self.min_(pack_winner_keys(dist_a, gid)))
        local = dist_keys(dist_a, gid < 0)
        gkey = self.min_(local.clone())
        ggid = self.min_(winner_index_candidates(local, gkey, gid))
        return winner_from_keys(gkey, ggid)

    def reduce_winners(self, dist_a: torch.Tensor, gid: torch.Tensor, rows: Optional[torch.Tensor] = None,
                       train_full: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """dist_a[m] local minima (NaN = this shard has no row of the class), gid[m] original
        index of the local winner.  Returns the global minimum distance, the global winner's original
        index and its trace on every rank: gathered from `train_full` (the replicated training set in
        original order) when given, else all-reduced from `rows[m, d]` (owner contributes, others
        zeros -> exact)."""
        gmin, ggid = self.reduce_winner_index(dist_a, gid)
        if train_full is not None:
            winners = train_full.index_select(0, ggid.clamp(min=0))
            winners = torch.where((ggid >= 0)[:, None], winners, torch.zeros_like(winners))
        else:
            mine = (ggid >= 0) & (gid.to(torch.int64) == ggid)
            winners = torch.where(mine[:, None], rows, torch.zeros_like(rows))
            self.sum_(winners)
        return gmin, ggid, winners

    def reduce_min_nan(self, d: torch.Tensor) -> torch.Tensor:
        """min over ranks where NaN means 'empty range on this shard' (+inf is a distance like any other)."""
        return keys_dist(self.min_(dist_keys(d)))

    # -- LSA: merge per-shard (max, sum) -------------------------------------------------------
    def reduce_lse(self, mx: torch.Tensor, sm: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        g = self.max_(mx.clone())
        scale = torch.where(torch.isinf(mx) & (mx < 0), torch.zeros_like(mx), torch.exp(mx - g))
        s = self.sum_((sm * scale).to(torch.float64))
        return g, s


# ------------------------------------------------------------------------------------------
# nearest-neighbour engine (DSA)
# ------------------------------------------------------------------------------------------
class NnEngine:
    def __init__(self, t_sorted: torch.Tensor, class_off: np.ndarray, t_gid: torch.Tensor, cap: Optional[int] = None,
                 seeds: bool = True):
        """t_sorted: [n, d] float32/float64 on the GPU, rows grouped by class (offsets class_off,
        ascending original index inside a class); t_gid[n] int32 original indices."""
        self.dev = require_cuda()
        self.lib = _lib.load()
        self.t = t_sorted.contiguous()
        self.n, self.d = self.t.shape
        self.dtype = tip_dtype(self.t.dtype)
        self.class_off = np.asarray(class_off, dtype=np.int64)
        self.num_classes = self.class_off.shape[0] - 1
        self.class_off_dev = torch.from_numpy(self.class_off.astype(np.int32)).to(self.dev)
        self.max_class_rows = int(np.diff(self.class_off).max()) if self.num_classes > 0 else 0
        self._q_off_dev = BoundedCache(65)
        self.t_gid = t_gid.to(torch.int32).contiguous()
        self.cap = int(cap) if cap else (DEFAULT_CAP if self.d <= 256 else DEFAULT_CAP_LONG)
        self.pitch = int(self.lib.tip_pair_pitch(self.d, 1))
        sms = C.c_int(0)
        _lib.check(self.lib.tip_device_info(C.byref(sms), None, None), "tip_device_info")
        self.sms = sms.value
        qt, tt = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.tip_nn_filter_tile(self.d, C.byref(qt), C.byref(tt)), "tip_nn_filter_tile")
        self.row_tile, self.col_tile = qt.value, tt.value
        self.resident = int(self.lib.tip_nn_filter_kind(self.d)) == 1     # resident-query kernel (short traces)
        self.stats = torch.zeros(2, dtype=torch.int64, device=self.dev)
        self._item_cache = BoundedCache(65)
        self._plans = BoundedCache(8)
        self._work = BoundedCache(16)
        self._inputs = BoundedCache(8)
        self.sched_counter = torch.zeros(2, dtype=torch.int32, device=self.dev)
        self.last_cand_cnt_by_mode = {}
        # N_train-sharded engines: the whole (post-subsample) training set in ORIGINAL row order, replicated on
        # every rank, from which the global stage-1 winners are gathered by index (set by the owner)
        self.t_full = None
        if self.n > 0:
            # Distances are translation invariant: the packed operands hold bf16(x - center).  For general traces the
            # global mean shrinks the rounding error; traces that are exactly representable in bf16 (bf16-stored
            # activations, BASELINE config 5) are packed LOSSLESSLY with center = 0 — centring would only create a
            # rounding error (at C5: 33 candidate chunks per query instead of ~3, and a 7 ms re-rank per pass).
            if self._bf16_exact(self.t):
                self.center = torch.zeros(self.d, dtype=torch.float32, device=self.dev)
            else:
                self.center = self.t.mean(dim=0, dtype=torch.float64).to(torch.float32).contiguous()
            self.t_pack = torch.empty((self.n, self.pitch), dtype=torch.bfloat16, device=self.dev)
            sq = torch.empty(self.n, dtype=torch.float32, device=self.dev)
            err = torch.empty(self.n, dtype=torch.float32, device=self.dev)
            _lib.check(self.lib.tip_pair_prep(_p(self.t), self.dtype, self.n, self.d, _p(self.center), _lib.ROLE_TRAIN,
                                              1, -2.0, 1.0, _p(self.t_pack), _p(sq), _p(err), _stream()), "tip_pair_prep")
            self.rmax = float(torch.sqrt(sq.max()).item()) * (1.0 + 1e-6)
            self.errmax = float(err.max().item()) * (1.0 + 1e-6)   # measured bf16 rounding of the train rows
        else:
            self.center = torch.zeros(self.d, dtype=torch.float32, device=self.dev)
            self.t_pack, self.rmax, self.errmax = None, 0.0, 0.0
        # The filter's window needs finite bounds on the packed train rows.  Rows beyond float32's range (float64
        # traces above ~3e38, or float32 ones whose squared norm overflows) have none: every query of such an engine
        # takes the re-rank's exact scan, which has no such limit.
        self.filter_ok = math.isfinite(self.rmax) and math.isfinite(self.errmax)
        # Stage-2 seeds (short traces / resident-query kernel, where the warm-up of the running minima costs ~15 % of
        # the filter): for every train row an upper bound on the distance to its nearest other-class row = the exact
        # distance to the nearest one inside a fixed stratified sample of the training set, found once at fit time
        # with this very engine machinery.
        self.seed_b = None
        if seeds and self.n >= 4096 and self.num_classes >= 2 and self.resident:
            self.seed_b = self._other_class_seeds()
        # Optional fit-time table (build_other_class_table): dist_b of surprise.py:622-631 depends on the test input
        # only through WHICH train row won stage 1, so it can be tabulated per train row once per training set.
        self.table_b = None

    def build_other_class_table(self, chunk_rows: int = 1 << 16) -> torch.Tensor:
        """For every train row the exact NumPy-order distance to its nearest row of another class (NaN when there is
        none): the second stage of DSA for any future winner, found with the same filter + re-rank as a scoring call.
        N_train x N_train pairs once per training set; a call then only runs stage 1 and looks dist_b up."""
        cls_of_row = np.repeat(np.arange(self.num_classes), np.diff(self.class_off)).astype(np.int32)
        table = torch.empty(self.n, dtype=self.t.dtype, device=self.dev)
        for s in range(0, self.n, chunk_rows):
            e = min(self.n, s + chunk_rows)
            q_off = (np.clip(self.class_off, s, e) - s).astype(np.int64)
            q_class = torch.from_numpy(cls_of_row[s:e]).to(self.dev)
            table[s:e] = self.search(self.t[s:e], q_class, q_off, _lib.RANGE_OTHER_CLASSES)[0]
        torch.cuda.current_stream().synchronize()
        self.table_b = table
        return table

    def _other_class_seeds(self, sample_rows: int = 8192) -> Optional[torch.Tensor]:
        step = max(1, self.n // sample_rows)
        pick = torch.arange(0, self.n, step, device=self.dev)
        cls_of_row = np.repeat(np.arange(self.num_classes), np.diff(self.class_off))
        sub_cls = cls_of_row[::step][:pick.shape[0]]
        sub_off = np.concatenate([[0], np.cumsum(np.bincount(sub_cls, minlength=self.num_classes))]).astype(np.int64)
        if np.count_nonzero(np.diff(sub_off)) < 2:
            return None
        sub = NnEngine(self.t.index_select(0, pick), sub_off, self.t_gid.index_select(0, pick), seeds=False)
        q_class = torch.from_numpy(cls_of_row.astype(np.int32)).to(self.dev)
        ub = sub.search(self.t, q_class, self.class_off, _lib.RANGE_OTHER_CLASSES)[0].to(torch.float32)
        ub = torch.where(torch.isnan(ub), torch.full_like(ub, float("inf")), ub).contiguous()
        torch.cuda.current_stream().synchronize()
        return ub

    @staticmethod
    def _bf16_exact(t: torch.Tensor, chunk_rows: int = 1 << 18) -> bool:
        """True if every trace value survives a round trip through bfloat16 (checked in row chunks)."""
        if t.dtype != torch.float32:
            return False
        for r0 in range(0, t.shape[0], chunk_rows):
            c = t[r0:r0 + chunk_rows]
            if not bool((c.to(torch.bfloat16).to(torch.float32) == c).all()):
                return False
        return True

    @classmethod
    def from_host(cls, train: np.ndarray, labels: np.ndarray, num_classes: int, gids: Optional[np.ndarray] = None,
                  cap: Optional[int] = None, seeds: bool = True) -> "NnEngine":
        dev = require_cuda()
        order, off = class_layout(labels, num_classes)
        t = to_device(train, dev)
        idx = torch.from_numpy(order).to(dev)
        gid = idx if gids is None else torch.from_numpy(np.asarray(gids)[order]).to(dev)
        if t.dtype not in (torch.float32, torch.float64):
            t = t.to(torch.float32)          # device-resident bf16 / fp16 traces: exact widening
        return cls(t.index_select(0, idx), off, gid, cap, seeds)

    def work_buffer(self, m: int, dtype: torch.dtype) -> torch.Tensor:
        """Scratch of tip_nn_rerank for m queries: zero-filled once, every call leaves it re-armed."""
        def make():
            nbytes = int(self.lib.tip_nn_rerank_work_bytes(m, tip_dtype(dtype)))
            return torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)

        return self._work.get_or_make((int(m), dtype), make)

    def input_buffer(self, rows: int, dtype: torch.dtype) -> torch.Tensor:
        """Persistent HBM landing buffer for a batch of `rows` test traces (the H2D target of
        DSA.__call__ and the gather source of the captured search)."""
        return self._inputs.get_or_make((int(rows), dtype),
                                        lambda: torch.zeros((rows, self.d), dtype=dtype, device=self.dev))

    def ranges(self, mode: int):
        off = self.class_off
        if mode == _lib.RANGE_SAME_CLASS:
            return [[(off[c], off[c + 1])] for c in range(self.num_classes)]
        return [[(0, off[c]), (off[c + 1], off[-1])] for c in range(self.num_classes)]

    def query_state(self, m: int):
        """Filter-side state of m queries: packed bf16 operand, |h|^2, rounding-error norm, running
        minimum bits, candidate count (what tip_nn_query_prep fills)."""
        return (torch.empty((m, self.pitch), dtype=torch.bfloat16, device=self.dev),
                torch.empty(m, dtype=torch.float32, device=self.dev),
                torch.empty(m, dtype=torch.float32, device=self.dev),
                torch.empty(m, dtype=torch.int32, device=self.dev),
                torch.empty(m, dtype=torch.int32, device=self.dev))

    def other_class_mixed(self, q_off: np.ndarray, m: int) -> bool:
        """Few queries per class: the other-class stage tiles across class boundaries (full tiles) and masks each
        query's own class; many: class-aligned tiles never touch their own class's rows."""
        populated = int(np.count_nonzero(np.diff(np.asarray(q_off))))
        return m < 2 * self.row_tile * max(1, populated)

    def distinct_ok(self, q_off: np.ndarray, m: int) -> bool:
        """True if DSA's stage 2 runs once per distinct stage-1 winner (dsa_distances): the resident-query filter on
        class-aligned tiles, and every class's winner bits fit tip_dsa_distinct_winners' shared memory."""
        return (self.resident and not self.other_class_mixed(q_off, m)
                and 0 <= int(self.lib.tip_dsa_distinct_smem_bytes(self.max_class_rows)) <= 48 * 1024)

    def distinct_winners(self, pos: torch.Tensor, q_off: np.ndarray):
        """Stage-1 winner positions of class-sorted inputs -> the stage-2 queries once per distinct winner
        (tip_dsa_distinct_winners): (rows, packed query state, slot_class, live_end, k, slot)."""
        m = pos.shape[0]
        q_off_dev = self._q_off_dev.get_or_make(np.asarray(q_off, dtype=np.int64).tobytes(),
                                                lambda: torch.from_numpy(np.asarray(q_off, dtype=np.int32)).to(self.dev))
        keep_for_capture(q_off_dev, self.seed_b)
        rows = torch.empty((m, self.d), dtype=self.t.dtype, device=self.dev)
        state = self.query_state(m)
        slot_class, live_end, slot = (torch.empty(m, dtype=torch.int32, device=self.dev) for _ in range(3))
        k = torch.empty(self.num_classes, dtype=torch.int32, device=self.dev)
        per_class = int(np.diff(np.asarray(q_off, dtype=np.int64)).max()) if m else 0
        q_pack, q_sq, q_err, row_min, cand_cnt = state
        _lib.check(self.lib.tip_dsa_distinct_winners(_p(pos), m, _p(q_off_dev), _p(self.class_off_dev), self.num_classes,
                                                     self.max_class_rows, max(1, -(-per_class // 32)), _p(self.t),
                                                     self.dtype, self.d, _p(self.center), _p(self.seed_b), self.rmax,
                                                     self.errmax, _p(rows), _p(q_pack), _p(q_sq), _p(q_err), _p(row_min),
                                                     _p(cand_cnt), _p(slot_class), _p(live_end), _p(k), _p(slot),
                                                     _stream()), "tip_dsa_distinct_winners")
        return rows, state, slot_class, live_end, k, slot

    def has_items(self, q_off: np.ndarray, mode: int) -> bool:
        """True if a search of this mode would launch the filter for queries with this class histogram."""
        if self.n == 0:
            return False
        ranges = self.ranges(mode)
        return any(int(q_off[c + 1]) > int(q_off[c]) and any(int(hi) > int(lo) for lo, hi in ranges[c])
                   for c in range(self.num_classes))

    def search(self, q: torch.Tensor, q_class: torch.Tensor, q_off: np.ndarray, mode: int, use_filter: bool = True,
               want_rows: bool = False, prepacked=None, next_query=None, q_idx: Optional[torch.Tensor] = None, fin=None,
               speculative: bool = False, live_end: Optional[torch.Tensor] = None):
        """q: [m, d] queries grouped by class (q_off), q_class[m] int32.  Returns, per query, the
        exact NumPy-order distance to its nearest train row in the range selected by `mode`
        (NaN when the range is empty on this shard), that row's position (-1 when empty), its
        original index, and (want_rows) a copy of the winning train rows.
        prepacked: query_state() already filled for q (by a previous search's next_query);
        next_query: query_state() to fill with the winning rows as the next search's queries.
        q_idx: int32 [m] — the queries are rows q_idx[r] of q (class-sorted order over the caller's buffer; no gathered
        copy); fin: (dist_a, gid, idx, n_total, out) — fused result scatter of DSA's last stage (tip_rerank_extras).
        speculative: queries whose candidate list is empty or overflowed are only counted in work_buffer(m)[0] (no
        exhaustive-scan launch); the caller checks overflow_count() and repeats the call without it if non-zero.
        live_end: int32 [m] (distinct_winners) — query rows at and past live_end[r] hold no query; the filter draws
        every item from its pool and skips the query tiles without live rows (tip_nn_filter_live)."""
        m = q.shape[0] if q_idx is None else q_idx.shape[0]
        use_filter = use_filter and self.filter_ok
        out_dist = torch.empty(m, dtype=q.dtype, device=self.dev)
        out_pos = torch.empty(m, dtype=torch.int32, device=self.dev)
        out_gid = torch.empty(m, dtype=torch.int32, device=self.dev)
        out_rows = torch.empty((m, self.d), dtype=q.dtype, device=self.dev) if want_rows else None
        if m == 0:
            return out_dist, out_pos, out_gid, out_rows
        lib = self.lib
        cand_idx = cand_cnt = None
        if use_filter and self.n > 0:
            ranges = self.ranges(mode)
            key = (mode, np.asarray(q_off, dtype=np.int64).tobytes(), live_end is not None)

            def make():            # host planning + upload once per (mode, class histogram)
                mixed = mode == _lib.RANGE_OTHER_CLASSES and self.other_class_mixed(q_off, m)
                if live_end is not None:
                    assert self.resident and not mixed
                    items, n_static = build_live_items(q_off, ranges, self.row_tile, self.col_tile), 0
                elif self.resident:
                    # resident-query kernel: one or two long items per CTA, equal tile counts
                    tiles = query_tiles(q_off, ranges, self.class_off, self.row_tile, mixed)
                    items, n_static = build_balanced_items(tiles, self.col_tile, self.sms, pool_frac=POOL_FRAC,
                                                           pool_tiles=POOL_TILES)
                else:
                    n_static = None
                    span_of = lambda pairs: span_tiles_for(pairs, self.sms)
                    if mixed:
                        items = build_other_class_items(q_off, self.class_off, self.row_tile, self.col_tile, span_of)
                    else:
                        pairs = count_tile_pairs(q_off, ranges, self.row_tile, self.col_tile)
                        items, _ = build_items(q_off, ranges, span_of(pairs), self.row_tile, self.col_tile)
                    items = span_major(items)
                flops = 2.0 * self.d * sum(int(q_off[c + 1] - q_off[c]) * sum(int(hi) - int(lo) for lo, hi in ranges[c])
                                           for c in range(self.num_classes))
                flagged = bool(items.shape[0] and (items[:, 5] & 1).any())
                n_static = items.shape[0] if n_static is None else n_static
                return (torch.from_numpy(items).to(self.dev) if items.shape[0] else None, items.shape[0], flops, flagged,
                        n_static)

            items_dev, n_items, flops, flagged, n_static = self._item_cache.get_or_make(key, make)
            if n_items > 0:
                if prepacked is not None:
                    q_pack, q_sq, q_err, row_min, cand_cnt = prepacked
                else:
                    q_pack, q_sq, q_err, row_min, cand_cnt = self.query_state(m)
                    _lib.check(lib.tip_nn_query_prep(_p(q), tip_dtype(q.dtype), m, self.d, _p(self.center), _p(q_pack),
                                                     _p(q_sq), _p(q_err), _p(row_min), _p(cand_cnt), _p(q_idx), _stream()),
                               "tip_nn_query_prep")
                cand_idx = torch.empty((m, self.cap, 2), dtype=torch.int32, device=self.dev)
                ev = None
                if PROFILE is not None:
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record()
                _lib.check(lib.tip_nn_filter_live(_p(q_pack), _p(q_sq), m, _p(self.t_pack), self.n, self.d, self.pitch,
                                                  _p(items_dev), n_items, _p(q_class if flagged else None),
                                                  _p(self.class_off_dev if flagged else None), self.rmax,
                                                  _p(q_err), self.errmax, _p(row_min), _p(cand_idx),
                                                  _p(cand_cnt), self.cap, n_static,
                                                  _p(self.sched_counter if n_static < n_items else None),
                                                  _p(live_end), _stream()), "tip_nn_filter_live")
                if ev is not None:
                    ev[1].record()
                    name = "nn_filter_same_class" if mode == _lib.RANGE_SAME_CLASS else "nn_filter_other_classes"
                    PROFILE.append((name, flops, ev[0], ev[1]))
        work = self.work_buffer(m, q.dtype)
        nq = [_p(t) for t in next_query] if next_query is not None else [None] * 5
        # stage 1 -> stage 2 hand-over: the winners' fit-time bounds seed the other-class search's running minima
        seed = self.seed_b if (next_query is not None and mode == _lib.RANGE_SAME_CLASS) else None
        keep_for_capture(work, self.sched_counter, self.t_pack, self.t, self.t_gid, self.class_off_dev, self.center,
                         items_dev if (use_filter and self.n > 0) else None, seed)
        ex = _lib.RerankExtras()
        ex.q_idx = 0 if q_idx is None else q_idx.data_ptr()
        ex.next_seed_ub = 0 if seed is None else seed.data_ptr()
        ex.next_t_rmax, ex.next_t_errmax = self.rmax, self.errmax
        ex.count_overflow_only = 1 if (speculative and cand_cnt is not None) else 0
        if fin is not None:
            f_a, f_gid, f_idx, f_n, f_out = fin
            ex.fin_dist_a, ex.fin_gid = f_a.data_ptr(), f_gid.data_ptr()
            ex.fin_idx = 0 if f_idx is None else f_idx.data_ptr()
            ex.fin_n_total, ex.fin_out = int(f_n), f_out.data_ptr()
        _lib.check(lib.tip_nn_rerank(_p(q), _p(self.t), tip_dtype(q.dtype), m, self.n, self.d, _p(cand_idx),
                                     _p(cand_cnt), self.cap, _p(q_class), _p(self.class_off_dev), self.num_classes,
                                     mode, _p(self.t_gid), _p(out_dist), _p(out_pos), _p(out_gid), _p(out_rows),
                                     _p(work), _p(self.stats),
                                     _p(self.center) if next_query is not None else None, *nq,
                                     C.byref(ex), _stream()),
                   "tip_nn_rerank")
        self.last_cand_cnt = cand_cnt
        if cand_cnt is not None:
            self.last_cand_cnt_by_mode[mode] = (cand_cnt, cand_idx)
        return out_dist, out_pos, out_gid, out_rows

    def gather(self, pos: torch.Tensor) -> torch.Tensor:
        return gather_rows(self.t, pos)


def gather_rows(src: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """src[pos] for int32 row positions `pos` (tip_gather_rows)."""
    out = torch.empty((pos.shape[0], src.shape[1]), dtype=src.dtype, device=src.device)
    if pos.shape[0]:
        _lib.check(_lib.load().tip_gather_rows(_p(src), src.shape[1] * src.element_size(), _p(pos), pos.shape[0],
                                               _p(out), _stream()), "tip_gather_rows")
    return out


def winner_queries(engine: "NnEngine", p2p: Optional[P2PExchange], gdist: Optional[torch.Tensor],
                   ggid: Optional[torch.Tensor], m: int, dtype: torch.dtype, state2):
    """Global stage-1 winners -> (dist_a, original index, winning rows) + the packed stage-2 query
    state, gathered from the replicated training set (tip_shard_winner_queries).  With `p2p` the
    per-shard records of the exchange started by the last push are reduced inside the kernel."""
    dev = engine.dev
    dist_a = torch.empty(m, dtype=dtype, device=dev)
    gid = torch.empty(m, dtype=torch.int32, device=dev)
    rows = torch.empty((m, engine.d), dtype=dtype, device=dev)
    q_pack, q_sq, q_err, row_min, cand_cnt = state2
    _lib.check(engine.lib.tip_shard_winner_queries(p2p.handle if p2p is not None else None, _p(gdist), _p(ggid),
                                                   tip_dtype(dtype), m, engine.d, _p(engine.t_full),
                                                   engine.t_full.shape[0], _p(engine.center), _p(dist_a), _p(gid), _p(rows),
                                                   _p(q_pack), _p(q_sq), _p(q_err), _p(row_min), _p(cand_cnt), _stream()),
               "tip_shard_winner_queries")
    return dist_a, gid, rows


def dsa_distances(engine: NnEngine, x: torch.Tensor, q_class: torch.Tensor, q_off: np.ndarray,
                  comm: Optional[TrainShardComm] = None, use_filter: bool = True, q_idx: Optional[torch.Tensor] = None,
                  scatter=None, speculative: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """surprise.py:615-631 for class-sorted queries x: (dist_a, dist_b, winner original index).
    Eager launches (the CUDA-graph plans below replay the same sequence).  Single shard only: q_idx — the
    class-sorted queries are rows q_idx[r] of x (the gather is fused into the pack and the re-rank); scatter =
    (idx, n_total, out) — the last re-rank also writes dist_a, dist_b, winner, dist_a / dist_b into out[4, n_total]."""
    sharded = comm is not None and comm.world > 1
    use_filter = use_filter and engine.filter_ok
    m = x.shape[0] if q_idx is None else q_idx.shape[0]
    if not sharded and engine.table_b is not None and engine.table_b.dtype == x.dtype:
        # fit-time table: stage 1 only, dist_b looked up by the winner's position
        dist_a, pos, gid, _ = engine.search(x, q_class, q_off, _lib.RANGE_SAME_CLASS, use_filter, q_idx=q_idx,
                                            speculative=speculative)
        found = pos >= 0
        dist_b = torch.where(found, engine.table_b.index_select(0, pos.clamp_min(0).to(torch.int64)),
                             torch.full_like(dist_a, float("nan")))
        if scatter is not None:
            pack_out(dist_a, dist_b, gid, scatter[0], scatter[2])
        return dist_a, dist_b, gid
    if not sharded:
        fuse = use_filter and engine.has_items(q_off, _lib.RANGE_OTHER_CLASSES)
        if fuse and engine.distinct_ok(q_off, m):
            # stage 2 depends on the input only through its stage-1 winner: search once per distinct winner (slots in
            # training-row order inside each class's range), then hand every input its slot's dist_b
            dist_a, pos, gid, _ = engine.search(x, q_class, q_off, _lib.RANGE_SAME_CLASS, use_filter, q_idx=q_idx,
                                                speculative=speculative)
            rows, state2, slot_class, live_end, _, slot = engine.distinct_winners(pos, q_off)
            slot_b = engine.search(rows, slot_class, q_off, _lib.RANGE_OTHER_CLASSES, use_filter, prepacked=state2,
                                   live_end=live_end, speculative=speculative)[0]
            dist_b = torch.empty_like(dist_a)
            idx, n_total, out = (None, 0, None) if scatter is None else scatter
            _lib.check(engine.lib.tip_dsa_slot_out(_p(slot_b), tip_dtype(slot_b.dtype), _p(slot), m, _p(dist_a), _p(gid),
                                                   _p(idx), int(n_total), _p(dist_b), _p(out), _stream()),
                       "tip_dsa_slot_out")
            return dist_a, dist_b, gid
        # single shard: stage 1's re-rank also emits its winners as the packed queries of stage 2
        state2 = engine.query_state(m) if fuse else None
        dist_a, _, gid, winners = engine.search(x, q_class, q_off, _lib.RANGE_SAME_CLASS, use_filter, want_rows=True,
                                                next_query=state2, q_idx=q_idx, speculative=speculative)
        fin = None if scatter is None else (dist_a, gid, scatter[0], scatter[1], scatter[2])
        dist_b = engine.search(winners, q_class, q_off, _lib.RANGE_OTHER_CLASSES, use_filter, prepacked=state2, fin=fin,
                               speculative=speculative)[0]
        return dist_a, dist_b, gid
    assert q_idx is None and scatter is None
    replica = engine.t_full is not None
    p2p = comm.p2p(engine.dev, m) if replica else None
    local_a, _, local_gid, local_rows = engine.search(x, q_class, q_off, _lib.RANGE_SAME_CLASS, use_filter,
                                                      want_rows=not replica)
    if replica:
        state2 = engine.query_state(m)
        if p2p is not None:
            p2p.push_nn(local_a, local_gid)
            dist_a, gid, winners = winner_queries(engine, p2p, None, None, m, x.dtype, state2)
        else:
            gmin, ggid = comm.reduce_winner_index(local_a, local_gid)
            dist_a, gid, winners = winner_queries(engine, None, gmin.contiguous(), ggid.to(torch.int32).contiguous(), m,
                                                  x.dtype, state2)
        prepacked = state2 if (use_filter and engine.has_items(q_off, _lib.RANGE_OTHER_CLASSES)) else None
    else:
        dist_a, gid, winners = comm.reduce_winners(local_a, local_gid, local_rows)
        prepacked = None
    local_b = engine.search(winners, q_class, q_off, _lib.RANGE_OTHER_CLASSES, use_filter, prepacked=prepacked)[0]
    if p2p is not None:
        p2p.push_nn(local_b, None)
        dist_b = torch.empty_like(local_b)
        p2p.min_into(dist_b)
    else:
        dist_b = comm.reduce_min_nan(local_b)
    return dist_a, dist_b, gid


def pack_out(dist_a: torch.Tensor, dist_b: torch.Tensor, gid: torch.Tensor, idx: Optional[torch.Tensor],
             out: torch.Tensor) -> None:
    """out[:, idx[r]] = (dist_a, dist_b, winner index, dist_a / dist_b) of class-sorted query r, as float64; the division
    runs in the dtype of dist_a and dist_b (tip_dsa_pack_out)."""
    _lib.check(_lib.load().tip_dsa_pack_out(_p(dist_a), _p(dist_b), tip_dtype(dist_a.dtype), _p(gid), _p(idx),
                                            gid.shape[0], out.shape[1], _p(out), _stream()), "tip_dsa_pack_out")


def reset_unscored(out: torch.Tensor, m: int) -> None:
    """A call that scores m < n_total rows leaves the others NaN / -1; which rows those are can change between calls."""
    if out.shape[1] != m:
        out.fill_(float("nan"))
        out[2].fill_(-1.0)


def dsa_scores(engine: NnEngine, x_in: torch.Tensor, idx: torch.Tensor, q_class: torch.Tensor, q_off: np.ndarray,
               out: torch.Tensor, comm: Optional[TrainShardComm] = None, use_filter: bool = True,
               speculative: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One DSA scoring call on the device, the sequence DsaPlan captures.  x_in: [n_total, d] test traces in the
    caller's row order; idx: int32 [m], the caller's row of every class-sorted query (classes by q_off, q_class[m]);
    out: float64 [4, n_total] <- dist_a, dist_b, winner index, dist_a / dist_b in the caller's order, NaN / -1 in the
    rows outside idx.  Returns dist_a, dist_b and the winner index in class-sorted order.  speculative: see
    NnEngine.search (single shard only)."""
    reset_unscored(out, idx.shape[0])
    if comm is None or comm.world <= 1:
        return dsa_distances(engine, x_in, q_class, q_off, None, use_filter, q_idx=idx,
                             scatter=(idx, out.shape[1], out), speculative=speculative)
    dist_a, dist_b, gid = dsa_distances(engine, gather_rows(x_in, idx), q_class, q_off, comm, use_filter)
    pack_out(dist_a, dist_b, gid, idx, out)
    return dist_a, dist_b, gid


class DsaPlan:
    """The whole scoring call for one (batch size, class histogram), `dsa_scores`, captured as CUDA graph(s).
    Inputs: `x_in` [n_total, d] (the engine's landing buffer for host uploads) and `idx` [m]
    (original row of every class-sorted query).  Output: `out` [4, n_total] float64 in the
    caller's order — dist_a, dist_b, winner index, dist_a / dist_b (divided in the trace dtype) —
    where rows the reference never scores keep NaN / -1.

    N_train sharded (comm.world > 1): with the peer-memory exchange the two exchange steps are
    kernels of ours and the call is still ONE graph; with the torch.distributed fallback the same steps run as
    three graph segments with one eager MIN all-reduce between consecutive segments (two for float64
    traces in the first exchange)."""

    def __init__(self, engine: "NnEngine", m: int, q_off: np.ndarray, dtype: torch.dtype, use_filter: bool,
                 comm: Optional[TrainShardComm] = None, n_total: Optional[int] = None):
        use_filter = use_filter and engine.filter_ok
        self.engine = engine
        self.q_off = np.asarray(q_off, dtype=np.int64).copy()
        dev = engine.dev
        self.m = int(m)
        self.n_total = int(m if n_total is None else n_total)
        self.x_in = engine.input_buffer(self.n_total, dtype)
        self.idx = torch.arange(self.m, dtype=torch.int32, device=dev)
        self.out = torch.full((4, self.n_total), float("nan"), dtype=torch.float64, device=dev)
        self.out[2].fill_(-1.0)
        self.out_host = torch.empty((4, self.n_total), dtype=torch.float64).pin_memory()
        self.idx_host = torch.empty(self.m, dtype=torch.int32).pin_memory()
        q_class = np.repeat(np.arange(engine.num_classes, dtype=np.int32), np.diff(self.q_off))
        self.q_class = torch.from_numpy(q_class).to(dev)
        self.comm = comm if (comm is not None and comm.world > 1) else None
        sharded = self.comm is not None
        if sharded and engine.t_full is None:
            raise RuntimeError("the sharded plan needs the replicated training set (NnEngine.t_full)")
        self.p2p = self.comm.p2p(dev, self.m) if sharded else None
        # Single shard with the filter on: the replayed graph has NO exhaustive-scan launches (two normally empty
        # launches per call); queries whose candidate list is empty or overflowed are only counted, and the caller
        # repeats such a call on the eager path (overflowed() / clear_overflow()).
        self.speculative = bool(use_filter and not sharded)
        self.overflow = engine.work_buffer(self.m, dtype)[:4].view(torch.int32)
        self.overflow_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        if not sharded or self.p2p is not None:
            def whole():
                dsa_scores(engine, self.x_in, self.idx, self.q_class, self.q_off, self.out, self.comm, use_filter,
                           self.speculative)

            segments = [(whole, True)]
        else:
            # torch.distributed fallback: static exchange buffers written by one graph segment,
            # all-reduced in place (eager), read by the next segment
            S = self.state = {}
            f32 = dtype == torch.float32
            # distances travel as dist_keys (integers, "no row" above +inf), so a real +inf survives the exchange
            S["keys"] = torch.zeros(self.m, dtype=torch.int64, device=dev)
            S["local"] = torch.zeros(self.m, dtype=torch.int64, device=dev)
            S["cand"] = torch.zeros(self.m, dtype=torch.int64, device=dev)
            S["bmin"] = torch.zeros(self.m, dtype=torch.int32 if f32 else torch.int64, device=dev)

            def seg_a():
                x = gather_rows(self.x_in, self.idx)
                la, _, lg, _ = engine.search(x, self.q_class, self.q_off, _lib.RANGE_SAME_CLASS, use_filter)
                S["lg"] = lg
                if f32:
                    S["keys"].copy_(pack_winner_keys(la, lg))
                else:
                    S["local"].copy_(dist_keys(la, lg < 0))
                    S["keys"].copy_(S["local"])

            def exch_1():
                self.comm.min_(S["keys"])
                if not f32:
                    S["cand"].copy_(winner_index_candidates(S["local"], S["keys"], S["lg"]))
                    self.comm.min_(S["cand"])

            def seg_b():
                if f32:
                    gmin, ggid = unpack_winner_keys(S["keys"])
                else:
                    gmin, ggid = winner_from_keys(S["keys"], S["cand"])
                state2 = engine.query_state(self.m)
                a, gid, winners = winner_queries(engine, None, gmin.contiguous(), ggid.to(torch.int32).contiguous(),
                                                 self.m, dtype, state2)
                S["a"], S["gid"] = a, gid
                pre = state2 if (use_filter and engine.has_items(self.q_off, _lib.RANGE_OTHER_CLASSES)) else None
                lb = engine.search(winners, self.q_class, self.q_off, _lib.RANGE_OTHER_CLASSES, use_filter, prepacked=pre)[0]
                S["bmin"].copy_(dist_keys(lb))

            def exch_2():
                self.comm.min_(S["bmin"])

            def seg_c():
                reset_unscored(self.out, self.m)
                pack_out(S["a"], keys_dist(S["bmin"]), S["gid"], self.idx, self.out)

            segments = [(seg_a, True), (exch_1, False), (seg_b, True), (exch_2, False), (seg_c, True)]

        self.steps, graphs, self._keep_alive = capture_graphs(segments, dev)
        self.graph = graphs[0] if len(segments) == 1 else None
        if self.speculative:
            self.overflow.zero_()     # whatever the warm-up ran on (a stale landing buffer) does not count

    def load_sorted(self, x_sorted: torch.Tensor):
        """Device-resident input already in class-sorted order (benchmarks, tools)."""
        assert self.n_total == self.m
        self.x_in.copy_(x_sorted)
        self.idx.copy_(torch.arange(self.m, dtype=torch.int32, device=self.idx.device))

    def run(self):
        for step in self.steps:
            step()
        return self.out

    def fetch_overflow(self):
        """enqueue the D2H copy of the overflow counter (speculative plans); read it with overflowed() after a sync"""
        if self.speculative:
            self.overflow_host.copy_(self.overflow, non_blocking=True)

    def overflowed(self) -> bool:
        return self.speculative and int(self.overflow_host[0]) != 0

    def clear_overflow(self):
        self.overflow.zero_()
        self.overflow_host.zero_()


def dsa_plan(engine: "NnEngine", m: int, q_off: np.ndarray, dtype: torch.dtype, use_filter: bool,
             comm: Optional[TrainShardComm] = None, n_total: Optional[int] = None) -> DsaPlan:
    n_total = int(m if n_total is None else n_total)
    key = (m, n_total, np.asarray(q_off, dtype=np.int64).tobytes(), dtype, use_filter, engine.cap, comm is not None,
           engine.table_b is not None)
    return engine._plans.get_or_make(key, lambda: DsaPlan(engine, m, q_off, dtype, use_filter, comm, n_total=n_total))


# ------------------------------------------------------------------------------------------
# Gaussian-KDE engine (LSA)
# ------------------------------------------------------------------------------------------
F16_NORM_SCALE = 64.0       # tail scale of the fp16 operand: |p|^2 / 2 / 64 must stay below 65504


class KdeEngine:
    def __init__(self, p_whitened, comm: Optional[TrainShardComm] = None):
        """p_whitened: [n, d] whitened, centred training traces: float64 on the host, or fp32 on the device (the
        device KDE fit's tip_whiten_dmma output; used in place).  With a communicator
        of more than one rank the engine keeps rows rank::world (N_train sharded) and merges the
        per-shard partial sums in log_kernel_sum (north_star: one exchange of partial KDE sums).

        Two packed operands are kept: the three-segment split-bf16 form (~2^-17 relative per product: always
        accurate enough for rtol 1e-4) and a one-segment fp16 form (11-bit significands, a third of the tensor
        work).  Which one a scoring call uses is decided by MEASURING the fast form's error on a sample of the
        queries (core/stable_kde.py)."""
        self.dev = require_cuda()
        self.lib = _lib.load()
        self.comm = comm if (comm is not None and comm.world > 1) else None
        if self.comm is not None:
            p_whitened = p_whitened[self.comm.rank::self.comm.world]
            if isinstance(p_whitened, np.ndarray):
                p_whitened = np.ascontiguousarray(p_whitened)
        self.n, self.d = p_whitened.shape
        self.precision = "split-bf16 x3 (h.h + h.l + l.h, ~2^-17 relative)"
        self.pitch = int(self.lib.tip_pair_pitch(self.d, 3))
        self.pitch1 = int(self.lib.tip_pair_pitch(self.d, 1))
        sms = C.c_int(0)
        _lib.check(self.lib.tip_device_info(C.byref(sms), None, None), "tip_device_info")
        self.sms = sms.value
        if isinstance(p_whitened, torch.Tensor):
            p32 = p_whitened.to(self.dev, torch.float32).contiguous()
        else:
            p32 = to_device(p_whitened.astype(np.float32), self.dev)
        self.t_pack = torch.empty((self.n, self.pitch), dtype=torch.bfloat16, device=self.dev)
        _lib.check(self.lib.tip_pair_prep(_p(p32), _lib.TIP_F32, self.n, self.d, None, _lib.ROLE_TRAIN, 3, 1.0, -0.5,
                                          _p(self.t_pack), None, None, _stream()), "tip_pair_prep")
        # fast form; unusable if a training value or its norm term leaves fp16's range
        self.t_pack_f16 = torch.empty((self.n, self.pitch1), dtype=torch.float16, device=self.dev)
        self.flags = torch.zeros(1, dtype=torch.int32, device=self.dev)
        _lib.check(self.lib.tip_pair_prep_f16(_p(p32), _lib.TIP_F32, self.n, self.d, None, _lib.ROLE_TRAIN, -0.5,
                                              F16_NORM_SCALE, _p(self.t_pack_f16), None, _p(self.flags), _stream()),
                   "tip_pair_prep_f16")
        torch.cuda.current_stream().synchronize()
        self.fast_ok = int(self.flags.item()) == 0 and self.comm is None
        if not self.fast_ok:
            self.t_pack_f16 = None
        self._items = BoundedCache(17)

    def _work_items(self, m: int):
        """Host planning + upload once per batch size."""
        def make():
            q_off = np.array([0, m], dtype=np.int64)
            ranges = [[(0, self.n)]]
            rt = int(self.lib.tip_kde_tile_rows())
            items, slots = build_items(q_off, ranges, span_tiles_for(count_tile_pairs(q_off, ranges, rt), self.sms), rt)
            items = span_major(items)
            # one partial per column part of a tile (tip_kde_slot_parts: 4 x 64 columns)
            return torch.from_numpy(items).to(self.dev), items.shape[0], slots * int(self.lib.tip_kde_slot_parts())

        return self._items.get_or_make(m, make)

    def log_kernel_sum(self, q: torch.Tensor, fast: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """q: [m, d] fp32 whitened, centred queries on the GPU.  Returns (mx, sm, qsq) with
        sum_i exp(-|p_i - q_j|^2/2) = exp(mx_j - qsq_j/2) * sm_j.  fast=True: the one-segment fp16 pass
        (sets flags[0] if a query leaves fp16's range)."""
        m = q.shape[0]
        lib = self.lib
        q_sq = torch.empty(m, dtype=torch.float32, device=self.dev)
        if fast:
            assert self.fast_ok
            q_pack = torch.empty((m, self.pitch1), dtype=torch.float16, device=self.dev)
            _lib.check(lib.tip_pair_prep_f16(_p(q), _lib.TIP_F32, m, self.d, None, _lib.ROLE_QUERY, 0.0, F16_NORM_SCALE,
                                             _p(q_pack), _p(q_sq), _p(self.flags), _stream()), "tip_pair_prep_f16")
        else:
            q_pack = torch.empty((m, self.pitch), dtype=torch.bfloat16, device=self.dev)
            _lib.check(lib.tip_pair_prep(_p(q), _lib.TIP_F32, m, self.d, None, _lib.ROLE_QUERY, 3, 1.0, 0.0, _p(q_pack),
                                         _p(q_sq), None, _stream()), "tip_pair_prep")
        items_dev, n_items, slots = self._work_items(m)
        keep_for_capture(items_dev, self.t_pack, self.t_pack_f16, self.flags)
        part_max = torch.full((slots, m), float("-inf"), dtype=torch.float32, device=self.dev)
        part_sum = torch.zeros((slots, m), dtype=torch.float32, device=self.dev)
        if fast:
            _lib.check(lib.tip_kde_lse_f16(_p(q_pack), m, _p(self.t_pack_f16), self.n, self.d, self.pitch1, _p(items_dev),
                                           n_items, _p(part_max), _p(part_sum), _stream()), "tip_kde_lse_f16")
        else:
            _lib.check(lib.tip_kde_lse(_p(q_pack), m, _p(self.t_pack), self.n, self.d, self.pitch, _p(items_dev),
                                       n_items, _p(part_max), _p(part_sum), _stream()), "tip_kde_lse")
        mx = torch.empty(m, dtype=torch.float32, device=self.dev)
        sm = torch.empty(m, dtype=torch.float32, device=self.dev)
        _lib.check(lib.tip_kde_combine(_p(part_max), _p(part_sum), m, slots, _p(mx), _p(sm), _stream()),
                   "tip_kde_combine")
        if self.comm is not None:
            p2p = self.comm.p2p(self.dev, m)
            mx, sm = p2p.lse(mx, sm) if p2p is not None else self.comm.reduce_lse(mx, sm)
        return mx, sm, q_sq


def whiten(x: torch.Tensor, cols: Optional[torch.Tensor], mu: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """(x[:, cols] - mu) @ w in fp32 on the GPU (scipy 1.4.1: points . cholesky(inv_cov))."""
    lib = _lib.load()
    m, d_in = x.shape
    d_out = w.shape[0]
    out = torch.empty((m, d_out), dtype=torch.float32, device=x.device)
    _lib.check(lib.tip_whiten(_p(x), tip_dtype(x.dtype), m, d_in, _p(cols), d_out, _p(mu), _p(w), _p(out), _stream()),
               "tip_whiten")
    return out


def quadratic_forms(x, centres: Sequence[Tuple[torch.Tensor, torch.Tensor]], cols: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q[k, j] = |(x_j - mu_k) . W_k|^2 for every (mu_k [d] float64, W_k [d, d] float32) pair: whitening on the
    GPU (tip_whiten, centred first) + a double-accumulated row norm (tip_row_sqnorm).  x: [m, d_in] device
    matrix (float32 / float64).  Returns float64 [len(centres), m] on the device."""
    lib = _lib.load()
    m = x.shape[0]
    out = torch.empty((len(centres), m), dtype=torch.float64, device=x.device)
    for k, (mu, w) in enumerate(centres):
        y = whiten(x, cols, mu, w)
        if m:
            _lib.check(lib.tip_row_sqnorm(_p(y), m, y.shape[1], _p(out[k]), _stream()), "tip_row_sqnorm")
    return out


# ------------------------------------------------------------------------------------------
# k-means discriminator of MultiModalSA (surprise.py:102-133): device k-means + silhouette
# ------------------------------------------------------------------------------------------
KMEANS_MAX_K = 64


def silhouette_items(counts: np.ndarray, span_tiles: int, row_tile: int = _lib.ROW_TILE,
                     col_tile: int = _lib.COL_TILE) -> Tuple[np.ndarray, np.ndarray]:
    """Work list of the silhouette pass over label-sorted rows (cluster c = rows [off[c], off[c+1])): every
    query tile x every span of columns inside ONE cluster, so that each partial-sum slot belongs to one
    cluster.  Returns (items [n, 6] in span-major order, slot_cluster [slots] int32, non-decreasing)."""
    counts = np.asarray(counts, dtype=np.int64)
    off = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=off[1:])
    n = int(off[-1])
    ranges = [[(int(off[c]), int(off[c + 1])) for c in range(len(counts)) if counts[c] > 0]]
    items, _ = build_items(np.array([0, n], dtype=np.int64), ranges, span_tiles, row_tile, col_tile)
    slots = int(items[:, 4].max()) + 1 if items.shape[0] else 0
    slot_cluster = np.zeros(slots, dtype=np.int32)
    slot_cluster[items[:, 4]] = np.searchsorted(off, items[:, 2], side="right") - 1
    return span_major(items), slot_cluster


def _device_sms(lib) -> int:
    sms = C.c_int(0)
    _lib.check(lib.tip_device_info(C.byref(sms), None, None), "tip_device_info")
    return sms.value


def kmeans_fit(x: torch.Tensor, k: int, n_init: int, max_iter: int, tol: float, seed: int):
    """All n_init runs of sklearn's KMeans(k, init="k-means++", algorithm="lloyd") on the [n, d] device matrix x
    (float32 / float64): one cooperative kernel for seeding + Lloyd, one predict launch for the final labels and
    inertia of every run.  Returns (centres [k, d] x.dtype, labels [n] int32, inertia, n_iter) of the run with
    the lowest inertia (ties: the lowest run), all but the two scalars on the device.  max_iter = 0 stops after
    the seeding: the centres are the k-means++ seeds and n_iter is 0."""
    if max_iter < 0 or tol < 0:
        raise ValueError("max_iter must be >= 0 and tol >= 0")
    lib = _lib.load()
    n, d = x.shape
    dt = tip_dtype(x.dtype)
    tol_abs = float(torch.var(x, dim=0, correction=0).mean()) * tol if tol > 0 else 0.0
    wb = int(lib.tip_kmeans_work_bytes(n, d, k, n_init, dt))
    if wb < 0:
        raise ValueError(f"k-means of {n} x {d} rows with k={k}, n_init={n_init} is not supported: "
                         f"{lib.tip_last_error().decode(errors='replace')}")
    work = torch.empty(wb, dtype=torch.uint8, device=x.device)
    cen = torch.empty((n_init, k, d), dtype=x.dtype, device=x.device)
    n_iter = torch.zeros(n_init, dtype=torch.int32, device=x.device)
    _lib.check(lib.tip_kmeans_fit(_p(x), dt, n, d, k, n_init, max_iter, tol_abs, seed & (2 ** 64 - 1), _p(work),
                                  _p(cen), _p(n_iter), _stream()), "tip_kmeans_fit")
    del work
    labels = torch.empty((n_init, n), dtype=torch.int32, device=x.device)
    sq = torch.empty((n_init, n), dtype=torch.float64, device=x.device)
    inertia = torch.empty(n_init, dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_kmeans_predict(_p(x), dt, n, d, _p(cen), k, n_init, _p(labels), _p(sq), _p(inertia), _stream()),
               "tip_kmeans_predict")
    inert = inertia.cpu().numpy()
    best = int(np.argmin(inert))          # first minimum: ties go to the lowest run
    return cen[best].clone(), labels[best].clone(), float(inert[best]), int(n_iter[best].item())


def kmeans_predict(x: torch.Tensor, centres: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Nearest centre of every row (ties: lowest index) and its squared distance (float64), on the device."""
    lib = _lib.load()
    n, d = x.shape
    centres = centres.to(device=x.device, dtype=x.dtype).contiguous()
    labels = torch.empty(n, dtype=torch.int32, device=x.device)
    sq = torch.empty(n, dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_kmeans_predict(_p(x), tip_dtype(x.dtype), n, d, _p(centres), centres.shape[0], 1, _p(labels),
                                      _p(sq), None, _stream()), "tip_kmeans_predict")
    return labels, sq


def _gmm_work(lib, n: int, d: int, k: int, scatter_chunks: int, dev) -> torch.Tensor:
    wb = int(lib.tip_gmm_work_bytes(n, d, k, scatter_chunks))
    if wb < 0:
        raise ValueError(f"Gaussian mixture of {n} x {d} rows with {k} components is not supported: "
                         f"{lib.tip_last_error().decode(errors='replace')}")
    return torch.empty(wb, dtype=torch.uint8, device=dev)


def gmm_quad(x: torch.Tensor, means: torch.Tensor, prec_chol: torch.Tensor) -> torch.Tensor:
    """q[k, i] = |(x_i - means_k) . prec_chol_k|^2 (float64 [K, n], fp64 tensor cores) for the [n, d] device matrix
    x (float32 / float64); means [K, d] and the upper-triangular prec_chol [K, d, d] are float64 on the device."""
    lib = _lib.load()
    n, d = x.shape
    k = means.shape[0]
    q = torch.empty((k, n), dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_gmm_quad(_p(x), tip_dtype(x.dtype), n, d, _p(means), _p(prec_chol), k, _p(q), _stream()),
               "tip_gmm_quad")
    return q


def gmm_log_det(prec_chol: torch.Tensor) -> torch.Tensor:
    """sklearn _compute_log_det_cholesky ('full'): sum of the logs of the factor's diagonal, per component."""
    return torch.log(torch.diagonal(prec_chol, dim1=1, dim2=2)).sum(dim=1)


def gmm_resp(q: torch.Tensor, d: int, log_weights: torch.Tensor, log_det: torch.Tensor, want_resp: bool = True,
             want_lse: bool = False, want_labels: bool = False, want_bound: bool = False, work=None):
    """E-step tail on q [K, n]: (resp [K, n], lse [n], labels [n] int64, lower bound [1]) on the device, each None
    unless asked for."""
    lib = _lib.load()
    k, n = q.shape
    dev = q.device
    resp = torch.empty((k, n), dtype=torch.float64, device=dev) if want_resp else None
    lse = torch.empty(n, dtype=torch.float64, device=dev) if want_lse else None
    labels = torch.empty(n, dtype=torch.int64, device=dev) if want_labels else None
    bound = torch.empty(1, dtype=torch.float64, device=dev) if want_bound else None
    if want_bound and work is None:
        work = _gmm_work(lib, n, d, k, 0, dev)
    _lib.check(lib.tip_gmm_resp(_p(q), n, d, k, _p(log_weights), _p(log_det), _p(resp), _p(lse), _p(labels), _p(bound),
                                _p(work), _stream()), "tip_gmm_resp")
    return resp, lse, labels, bound


def gmm_moments(x: torch.Tensor, resp: torch.Tensor, work=None):
    """(nk [K], resp^T x [K, d], means [K, d]), float64 on the device (sklearn _estimate_gaussian_parameters)."""
    lib = _lib.load()
    n, d = x.shape
    k = resp.shape[0]
    if work is None:
        work = _gmm_work(lib, n, d, k, 0, x.device)
    nk = torch.empty(k, dtype=torch.float64, device=x.device)
    sums = torch.empty((k, d), dtype=torch.float64, device=x.device)
    means = torch.empty((k, d), dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_gmm_moments(_p(x), tip_dtype(x.dtype), n, d, _p(resp), k, _p(nk), _p(sums), _p(means), _p(work),
                                   _stream()), "tip_gmm_moments")
    return nk, sums, means


def gmm_scatter(x: torch.Tensor, resp: torch.Tensor, means: torch.Tensor, nk: Optional[torch.Tensor] = None,
                reg_covar: float = 0.0, scatter_chunks: int = 0, work=None) -> torch.Tensor:
    """[K, d, d] float64: the weighted scatter matrices S_k (nk None) or the covariances S_k / nk + reg_covar I.
    scatter_chunks: row chunks of the reduction (0: the library's choice; see gmm_scatter_chunks)."""
    lib = _lib.load()
    n, d = x.shape
    k = resp.shape[0]
    if work is None:
        work = _gmm_work(lib, n, d, k, scatter_chunks, x.device)
    out = torch.empty((k, d, d), dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_gmm_scatter(_p(x), tip_dtype(x.dtype), n, d, _p(resp), _p(means), k, _p(nk), float(reg_covar),
                                   int(scatter_chunks), _p(out), _p(work), _stream()), "tip_gmm_scatter")
    return out


def gmm_scatter_chunks(n: int, d: int, k: int, requested: int = 0) -> int:
    """Row chunks tip_gmm_scatter uses for this shape (requested 0: automatic), after the scratch cap."""
    return int(_lib.load().tip_gmm_scatter_chunks(n, d, k, requested))


GMM_FIT_ERROR = ("Fitting the mixture model failed because some components have ill-defined empirical covariance "
                 "(for instance caused by singleton or collapsed samples). Try to decrease the number of components, "
                 "increase reg_covar, or scale the input data.")


def gmm_factor(cov: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """sklearn _compute_precision_cholesky ('full') on the device, batched over the components, float64:
    prec_chol_k = inv(cholesky(cov_k))^T (upper triangular).  Returns (prec_chol [K, d, d], log det [K], info [K]
    int32: non-zero where cov_k is not positive definite; the caller raises)."""
    chol, info = torch.linalg.cholesky_ex(cov)
    eye = torch.eye(cov.shape[-1], dtype=cov.dtype, device=cov.device).expand_as(cov)
    prec = torch.linalg.solve_triangular(chol, eye, upper=False).transpose(1, 2).contiguous()
    return prec, gmm_log_det(prec), info


def gmm_init(x: torch.Tensor, labels: torch.Tensor, k: int, reg_covar: float, work=None):
    """sklearn GaussianMixture._initialize from hard labels (one-hot responsibilities, weights = nk / n).
    Returns (weights, means, covariances, prec_chol, log_det, info) on the device."""
    if work is None:
        work = _gmm_work(_lib.load(), x.shape[0], x.shape[1], k, 0, x.device)
    resp = torch.nn.functional.one_hot(labels.to(torch.int64), k).to(torch.float64).t().contiguous()
    nk, _, means = gmm_moments(x, resp, work)
    cov = gmm_scatter(x, resp, means, nk, reg_covar, 0, work)
    prec, log_det, info = gmm_factor(cov)
    return nk / x.shape[0], means, cov, prec, log_det, info


def _raise_if_failed(info: torch.Tensor, bound: Optional[torch.Tensor] = None):
    flags = info.to(torch.float64) if bound is None else torch.cat([info.to(torch.float64), bound])
    h = flags.cpu().numpy()
    if np.any(h[:info.shape[0]] != 0) or (bound is not None and not np.isfinite(h[-1])):
        raise ValueError(GMM_FIT_ERROR)
    return None if bound is None else float(h[-1])


def _gmm_step(x, weights, means, prec_chol, log_det, reg_covar, work, ev=None):
    """One E-step + M-step on device state; returns (bound tensor [1], weights, means, cov, prec, log_det, info)."""
    d = x.shape[1]
    mark = (lambda i: ev[i].record()) if ev is not None else (lambda i: None)
    mark(0)
    q = gmm_quad(x, means, prec_chol)
    resp, _, _, bound = gmm_resp(q, d, torch.log(weights), log_det, want_bound=True, work=work)
    mark(1)
    nk, sums, new_means = gmm_moments(x, resp, work)
    weights = nk / nk.sum()
    cov = gmm_scatter(x, resp, new_means, nk, reg_covar, 0, work)
    mark(2)
    prec, new_log_det, info = gmm_factor(cov)
    mark(3)
    return bound, weights, new_means, cov, prec, new_log_det, info


def gmm_em_step(x: torch.Tensor, weights: torch.Tensor, means: torch.Tensor, prec_chol: torch.Tensor,
                reg_covar: float):
    """One sklearn EM iteration (_e_step + _m_step) on the [n, d] device matrix x from the given float64 device
    state: returns (lower_bound of the E-step, weights, means, covariances, prec_chol) after the M-step.  Raises
    sklearn's ValueError when a covariance is not positive definite or the bound is not finite."""
    k = means.shape[0]
    work = _gmm_work(_lib.load(), x.shape[0], x.shape[1], k, 0, x.device)
    prec_chol = prec_chol.contiguous()
    bound, w, mu, cov, prec, _, info = _gmm_step(x, weights.contiguous(), means.contiguous(), prec_chol,
                                                 gmm_log_det(prec_chol), reg_covar, work)
    lb = _raise_if_failed(info, bound)
    return lb, w, mu, cov, prec


def gmm_fit(x: torch.Tensor, k: int, max_iter: int = 100, tol: float = 1e-3, reg_covar: float = 1e-6,
            seed: int = 0, timing: Optional[dict] = None) -> dict:
    """sklearn GaussianMixture(n_components=k, covariance_type="full", init_params="kmeans", n_init=1).fit on the
    [n, d] device matrix x: initial responsibilities from the labels of kmeans_fit(x, k, 1, 300, 1e-4, seed), then
    EM until |lower bound change| < tol or max_iter iterations.  One read-back per iteration (the bound and the
    factorisation flags).  Returns a dict of device tensors (weights, means, covariances, prec_chol, log_det) and
    host values (labels_init on the device, n_iter, converged, lower_bound, lower_bounds).
    timing: a dict that receives CUDA-event milliseconds per phase (kmeans, estep, mstep, factor, total)."""
    lib = _lib.load()
    n, d = x.shape
    work = _gmm_work(lib, n, d, k, 0, x.device)
    ev = None
    if timing is not None:
        new = lambda: torch.cuda.Event(enable_timing=True)
        t_start, t_km = new(), new()
        t_start.record()
    _, labels, _, _ = kmeans_fit(x, k, 1, 300, 1e-4, seed)
    if timing is not None:
        t_km.record()
    weights, means, cov, prec, log_det, info = gmm_init(x, labels, k, reg_covar, work)
    _raise_if_failed(info)
    steps = []
    lower_bound, bounds, converged, n_iter = -np.inf, [], False, 0
    for n_iter in range(1, max_iter + 1):
        prev = lower_bound
        if timing is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            steps.append(ev)
        bound, weights, means, cov, prec, log_det, info = _gmm_step(x, weights, means, prec, log_det, reg_covar, work, ev)
        lower_bound = _raise_if_failed(info, bound)
        bounds.append(lower_bound)
        if abs(lower_bound - prev) < tol:
            converged = True
            break
    if timing is not None:
        t_end = torch.cuda.Event(enable_timing=True)
        t_end.record()
        torch.cuda.synchronize()
        timing["kmeans"] = timing.get("kmeans", 0.0) + t_start.elapsed_time(t_km)
        for key, i in (("estep", 0), ("mstep", 1), ("factor", 2)):
            timing[key] = timing.get(key, 0.0) + sum(e[i].elapsed_time(e[i + 1]) for e in steps)
        timing["total"] = timing.get("total", 0.0) + t_start.elapsed_time(t_end)
    return {"weights": weights, "means": means, "covariances": cov, "prec_chol": prec, "log_det": log_det,
            "labels_init": labels, "n_iter": n_iter, "converged": converged, "lower_bound": lower_bound,
            "lower_bounds": bounds}


# ------------------------------------------------------------------------------------------
# MDSA's EmpiricalCovariance (surprise.py:374-393): location, scatter, pseudo-inverse
# ------------------------------------------------------------------------------------------
def cov_location(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(location [d] x.dtype = NumPy's x.mean(0) bit for bit, np.cov's float64 centring mean [d], non-finite flags
    [1] int32: bit 0 NaN, bit 1 inf) of the [n, d] device matrix x, all on the device."""
    lib = _lib.load()
    n, d = x.shape
    loc = torch.empty(d, dtype=x.dtype, device=x.device)
    mean = torch.empty(d, dtype=torch.float64, device=x.device)
    flags = torch.empty(1, dtype=torch.int32, device=x.device)
    _lib.check(lib.tip_cov_location(_p(x), tip_dtype(x.dtype), n, d, _p(loc), _p(mean), _p(flags), _stream()),
               "tip_cov_location")
    return loc, mean, flags


def cov_fit(x: torch.Tensor, timing: Optional[dict] = None) -> dict:
    """sklearn EmpiricalCovariance().fit on the [n, d] device matrix x (float32 / float64), n >= 1:
    - location = x.mean(0) in x's dtype (bit for bit), covariance = np.cov(x.T, bias=1) in float64: the DMMA
      scatter of tip_gmm_scatter (k = 1, unit weights) centred on the float64 mean, divided by n;
    - live columns: those with a non-zero diagonal.  A column whose centred values are all exactly 0 has an exactly
      zero row and column; it is left out of the eigendecomposition (its eigenvalue, 0, is one scipy drops too);
    - precision = scipy's pinvh of the live block: torch.linalg.eigh in float64, eigenvalues kept where
      |s| > d * eps * max|s| (d: all columns), (U / s) @ U^T; zero on dead rows and columns;
    - the scoring factor W [d_live, d_live] float32 = U diag(s^-1/2) over the kept s > 0 (zero columns after them),
      so that |(x[:, live] - location[live]) . W|^2 is the Mahalanobis form of the precision.
    Raises sklearn's ValueError on NaN / inf input (one read-back).  Returns device tensors: location, mean,
    covariance, live (int64), eigenvalues (of the live block), rank (host int), precision, score_mu (float64
    location[live]), score_w (None when d_live == 0).  timing: receives CUDA-event milliseconds (cov_location,
    scatter, eigh, total)."""
    n, d = x.shape
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timing is not None else None
    if ev:
        ev[0].record()
    loc, mean, flags = cov_location(x)
    if ev:
        ev[1].record()
    f = int(flags.item())
    if f & 1:
        raise ValueError("Input X contains NaN.")
    if f & 2:
        raise ValueError(f"Input X contains infinity or a value too large for {np.dtype(NP_DTYPE[x.dtype])!r}.")
    ones = torch.ones((1, n), dtype=torch.float64, device=x.device)
    nk = torch.full((1,), float(n), dtype=torch.float64, device=x.device)
    cov = gmm_scatter(x, ones, mean.reshape(1, d), nk, 0.0)[0]
    if ev:
        ev[2].record()
    live = torch.nonzero(torch.diagonal(cov) != 0).flatten()
    dl = int(live.shape[0])
    precision = torch.zeros((d, d), dtype=torch.float64, device=x.device)
    score_w, rank = None, 0
    s = torch.empty(0, dtype=torch.float64, device=x.device)
    if dl:
        s, u = torch.linalg.eigh(cov.index_select(0, live).index_select(1, live))
        cutoff = d * np.finfo(np.float64).eps * s.abs().max()
        keep = s.abs() > cutoff
        uk, sk = u[:, keep], s[keep]
        rank = int(sk.shape[0])
        block = (uk * (1.0 / sk)) @ uk.t()
        precision[live.unsqueeze(1), live.unsqueeze(0)] = block
        pos = sk > 0
        score_w = torch.zeros((dl, dl), dtype=torch.float32, device=x.device)
        score_w[:, :int(pos.sum())] = (uk[:, pos] * sk[pos].rsqrt()).to(torch.float32)
    if ev:
        ev[3].record()
        torch.cuda.synchronize()
        for key, i in (("cov_location", 0), ("scatter", 1), ("eigh", 2)):
            timing[key] = timing.get(key, 0.0) + ev[i].elapsed_time(ev[i + 1])
        timing["total"] = timing.get("total", 0.0) + ev[0].elapsed_time(ev[3])
    return {"location": loc, "mean": mean, "covariance": cov, "live": live, "eigenvalues": s, "rank": rank,
            "precision": precision, "score_mu": mean.new_empty(0) if not dl else
            loc.index_select(0, live).to(torch.float64), "score_w": score_w}


def cov_scores(x: torch.Tensor, fit: dict) -> torch.Tensor:
    """Squared Mahalanobis distances [m] (float64, device) of the rows of x to a cov_fit: fp32 whitening of the
    live columns (tip_whiten) + double row norms; zeros when no column is live."""
    if fit["score_w"] is None:
        return torch.zeros(x.shape[0], dtype=torch.float64, device=x.device)
    cols = fit["live"].to(torch.int32)
    return quadratic_forms(x, [(fit["score_mu"], fit["score_w"])], cols)[0]


# ------------------------------------------------------------------------------------------
# LSA's fit (surprise.py:417-437 + StableGaussianKDE, stable_kde.py:20-77): column variances, KDE fit
# ------------------------------------------------------------------------------------------
def col_var(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(var [d] x.dtype = np.var(x, axis=0) bit for bit, float64 column mean [d], non-finite flags [1] int32: bit 0
    NaN, bit 1 inf) of the [n, d] device matrix x, all on the device."""
    lib = _lib.load()
    n, d = x.shape
    var = torch.empty(d, dtype=x.dtype, device=x.device)
    mean = torch.empty(d, dtype=torch.float64, device=x.device)
    flags = torch.empty(1, dtype=torch.int32, device=x.device)
    _lib.check(lib.tip_col_var(_p(x), tip_dtype(x.dtype), n, d, _p(var), _p(mean), _p(flags), _stream()),
               "tip_col_var")
    return var, mean, flags


def whiten_f64(x: torch.Tensor, cols: Optional[torch.Tensor], mu: torch.Tensor, w_lower: torch.Tensor) -> torch.Tensor:
    """(x[:, cols] - mu) @ w_lower as fp32 [m, d'], accumulated in float64 on the fp64 tensor cores (tip_whiten_dmma);
    cols int32 [d'] or None, mu float64 [d'], w_lower float64 [d', d'] lower triangular."""
    lib = _lib.load()
    m, d_in = x.shape
    d = w_lower.shape[0]
    out = torch.empty((m, d), dtype=torch.float32, device=x.device)
    _lib.check(lib.tip_whiten_dmma(_p(x), tip_dtype(x.dtype), m, d_in, _p(cols), d, _p(mu), _p(w_lower), _p(out),
                                   _stream()), "tip_whiten_dmma")
    return out


KDE_MAX_INCREMENT = 1e-5
KDE_NOT_FIXED = ("Was not able to fix numerical imprecision in covariance matrix."
                 "Failing silently. All likelihoods will be reported as 0.")


def kde_cov_fact(n: int) -> float:
    """np.cov(X, bias=False, aweights=ones(n)/n)'s normalisation, with np.cov's own expressions (warning as np.cov
    does when it is not positive): fact = w_sum - ddof * sum(w * aweights) / w_sum, ddof = 1."""
    import warnings

    w = np.ones(n) / n
    w_sum = np.broadcast_to(w, (1, n)).sum(axis=1, dtype=np.float64)[0]      # np.average's scl
    fact = w_sum - 1 * np.sum(w * w) / w_sum
    if fact <= 0:
        warnings.warn("Degrees of freedom <= 0 for slice", RuntimeWarning, stacklevel=3)
        fact = 0.0
    return fact


def kde_fit(x: torch.Tensor, cols: Optional[np.ndarray] = None, mean: Optional[torch.Tensor] = None,
            timing: Optional[dict] = None) -> dict:
    """StableGaussianKDE(x[:, cols].T)'s fit (scott bandwidth, uniform weights) on the [n, D] device matrix x
    (float32 / float64), in float64 on the device:
    - covariance: np.cov(bias=False, aweights=1/n) = the DMMA scatter of tip_gmm_scatter (k = 1, resp = 1/n) of the
      kept columns (one index_select), centred on their float64 column mean (`mean` [D], from col_var, or computed
      here), times np.true_divide(1, fact) with np.cov's fact;
    - the stabilisation loop: while some eigenvalue (eigvalsh) of cov * factor^2 is <= d' eps max|lambda|, the
      diagonal is REPLACED by 1e-10 * 2^k; past 1e-5 the fit fails silently (prepare_failed, warning);
    - inv (inv_ex: a singular matrix sets prepare_failed), cholesky(2 pi covariance) for log_det, det for
      _norm_factor, W = cholesky(inv_cov) (cholesky_ex: failure raises NumPy's LinAlgError);
    - p = (x[:, cols] - mu) @ W as fp32 (tip_whiten_dmma), the operand of KdeEngine.
    A non-finite covariance raises LinAlgError("Eigenvalues did not converge"), as the host's eigh does.  Returns a
    dict of device tensors (rows = x[:, cols], covariance (unscaled, stabilised), inv (of it), whitening, mean [d'],
    p) and host values (diag_w, the whitening's diagonal, n, d, factor, rounds, prepare_failed, log_det,
    norm_factor); a failed fit has none of the entries from covariance on.  timing: receives CUDA-event milliseconds
    (col_var (when mean is None), scatter, factor, whiten, total) and the read-back count."""
    import warnings

    n, width = x.shape
    dev = x.device
    cols_t = None if cols is None else torch.from_numpy(np.ascontiguousarray(cols, dtype=np.int64)).to(dev)
    d = width if cols is None else int(cols_t.shape[0])
    marks = {}

    def mark(key):
        if timing is not None:
            marks[key] = torch.cuda.Event(enable_timing=True)
            marks[key].record()

    mark("start")
    if mean is None:
        _, mean, _ = col_var(x)
        mark("col_var")
    xs = x if cols_t is None else x.index_select(1, cols_t)
    mu = mean if cols_t is None else mean.index_select(0, cols_t)
    mu = mu.contiguous()
    resp = torch.full((1, n), 1.0 / n, dtype=torch.float64, device=dev)        # np.ones(n) / n
    inv_fact = float(np.true_divide(1, kde_cov_fact(n)))
    cov = gmm_scatter(xs.contiguous(), resp, mu.reshape(1, d))[0] * inv_fact
    mark("scatter")
    w = np.ones(n) / n
    neff = 1.0 / np.sum(w ** 2)
    factor = float(np.power(neff, -1.0 / (d + 4)))
    f2 = factor ** 2
    eps = np.finfo(np.float64).eps
    increment, rounds, failed, reads = 1e-10, 0, False, 0
    while True:
        try:
            lam = torch.linalg.eigvalsh(cov * f2)
        except torch.linalg.LinAlgError:             # e.g. NaN / inf entries: NumPy's eigh raises this
            raise np.linalg.LinAlgError("Eigenvalues did not converge") from None
        thr = d * eps * lam.abs().max()
        state = torch.stack([(lam <= thr).any().to(torch.float64), torch.isfinite(cov).all().to(torch.float64)]).cpu()
        rounds, reads = rounds + 1, reads + 1
        if state[1] == 0:
            raise np.linalg.LinAlgError("Eigenvalues did not converge")
        if state[0] == 0:
            break
        cov.fill_diagonal_(increment)
        if increment > KDE_MAX_INCREMENT:
            warnings.warn(KDE_NOT_FIXED)
            failed = True
            break
        increment += increment
    out = {"n": n, "d": d, "factor": factor, "rounds": rounds, "prepare_failed": failed, "mean": mu, "rows": xs}
    if failed:
        mark("factor")
        _finish_timing(timing, marks, reads)
        return out
    inv, info_inv = torch.linalg.inv_ex(cov)
    covariance = cov * f2
    inv_cov = inv / f2
    chol, info_c = torch.linalg.cholesky_ex(covariance * 2 * np.pi)
    log_det = 2 * torch.log(torch.diagonal(chol)).sum()
    norm_factor = torch.sqrt(torch.linalg.det(2 * np.pi * covariance))
    wl, info_w = torch.linalg.cholesky_ex(inv_cov)
    wl = wl.contiguous()                           # row-major, as the kernels and the query whitening read it
    diag_w = torch.diagonal(wl)
    host = torch.cat([torch.stack([info_inv.to(torch.float64), info_c.to(torch.float64), info_w.to(torch.float64),
                                   log_det, norm_factor]), diag_w]).cpu().numpy()
    reads += 1
    mark("factor")
    if host[0] != 0:                               # np.linalg.inv raised LinAlgError: the host sets prepare_failed
        out["prepare_failed"] = True
        _finish_timing(timing, marks, reads)
        return out
    if host[1] != 0 or host[2] != 0:
        raise np.linalg.LinAlgError("Matrix is not positive definite")
    cols32 = None if cols_t is None else cols_t.to(torch.int32)
    p = whiten_f64(x, cols32, mu, wl)
    mark("whiten")
    _finish_timing(timing, marks, reads)
    out.update({"covariance": cov, "inv": inv, "whitening": wl, "p": p, "diag_w": host[5:],
                "log_det": float(host[3]), "norm_factor": float(host[4])})
    return out


def _finish_timing(timing: Optional[dict], marks: dict, reads: int):
    if timing is None:
        return
    marks["end"] = torch.cuda.Event(enable_timing=True)
    marks["end"].record()
    torch.cuda.synchronize()
    keys = list(marks)
    for a, b in zip(keys[:-2], keys[1:-1]):
        timing[b] = timing.get(b, 0.0) + marks[a].elapsed_time(marks[b])
    timing["total"] = timing.get("total", 0.0) + marks["start"].elapsed_time(marks["end"])
    timing["reads"] = timing.get("reads", 0) + reads


def silhouette_samples(x: torch.Tensor, labels: torch.Tensor, n_clusters: int,
                       span_tiles: Optional[int] = None) -> torch.Tensor:
    """sklearn silhouette_samples of the [n, d] device matrix x (float32 / float64) under labels in
    [0, n_clusters) (every cluster non-empty): label-sorted, packed once in both roles, one wgmma pass of
    per-(row, cluster span) distance sums, one finishing kernel.  Returns float64 [n] in x's row order.
    span_tiles: column tiles per work-item span (None: span_tiles_for's choice for this card), so that a test can
    run the 1- and 16-tile layouts on any card."""
    lib = _lib.load()
    n, d = x.shape
    lab = labels.to(torch.int64)
    order = torch.argsort(lab, stable=True)
    counts = torch.bincount(lab, minlength=n_clusters)
    counts_h = counts.cpu().numpy()
    order32 = order.to(torch.int32)
    lab_sorted = lab.index_select(0, order).to(torch.int32)
    counts32 = counts.to(torch.int32)
    center = x.mean(dim=0).to(torch.float32)
    pitch = int(lib.tip_pair_pitch(d, 3))
    q_pack = torch.empty((n, pitch), dtype=torch.bfloat16, device=x.device)
    t_pack = torch.empty((n, pitch), dtype=torch.bfloat16, device=x.device)
    sq = torch.empty(n, dtype=torch.float32, device=x.device)
    _lib.check(lib.tip_sil_prep(_p(x), tip_dtype(x.dtype), n, d, _p(center), _p(order32), _p(q_pack), _p(t_pack),
                                _p(sq), _stream()), "tip_sil_prep")
    if span_tiles is None:
        pairs = math.ceil(n / _lib.ROW_TILE) * math.ceil(n / _lib.COL_TILE)
        span_tiles = span_tiles_for(pairs, _device_sms(lib))
    items, slot_cluster = silhouette_items(counts_h, span_tiles)
    slots = slot_cluster.shape[0]
    items_dev = torch.from_numpy(items).to(x.device)
    slot_dev = torch.from_numpy(slot_cluster).to(x.device)
    part = torch.zeros((slots, n), dtype=torch.float32, device=x.device)
    _lib.check(lib.tip_sil_dsum(_p(q_pack), _p(t_pack), _p(sq), n, d, pitch, _p(items_dev), items.shape[0], _p(part),
                                _stream()), "tip_sil_dsum")
    out = torch.empty(n, dtype=torch.float64, device=x.device)
    _lib.check(lib.tip_sil_finish(_p(part), n, slots, _p(slot_dev), _p(lab_sorted), _p(counts32), _p(order32), _p(out),
                                  _stream()), "tip_sil_finish")
    return out


LEV_MAX_LEN = 255         # distances are stored as uint8


def check_word_lengths(words: Sequence[str]) -> np.ndarray:
    """int64 code-point lengths of words; ValueError naming the first word longer than LEV_MAX_LEN."""
    lengths = np.fromiter(map(len, words), dtype=np.int64, count=len(words))
    too_long = np.flatnonzero(lengths > LEV_MAX_LEN)
    if too_long.size:
        k = int(too_long[0])
        raise ValueError(f"word {k} has {int(lengths[k])} code points; Levenshtein distances are stored as uint8, "
                         f"so words are limited to {LEV_MAX_LEN}")
    return lengths


def encode_words(words: Sequence[str]) -> Tuple[np.ndarray, np.ndarray]:
    """(ids int32, offsets int32 [len(words) + 1]) of a word list for tip_levenshtein: one id per Unicode code point
    (as Python's len counts them), numbered by descending frequency (ties by code point), so that the most common
    ones get the kernel's shared-memory match masks.  Raises ValueError, naming the first such word, when a word is
    longer than LEV_MAX_LEN code points: its distances would not fit the uint8 matrix."""
    lengths = check_word_lengths(words)
    offsets = np.zeros(len(words) + 1, dtype=np.int64)
    np.cumsum(lengths, out=offsets[1:])
    if offsets[-1] >= 2 ** 31:
        raise ValueError("the words have 2^31 code points or more; tip_levenshtein indexes them with int32")
    cps = np.frombuffer("".join(words).encode("utf-32-le", "surrogatepass"), dtype="<u4")
    uniq, inverse, counts = np.unique(cps, return_inverse=True, return_counts=True)
    rank = np.empty(uniq.shape[0], dtype=np.int32)
    rank[np.lexsort((uniq, -counts))] = np.arange(uniq.shape[0], dtype=np.int32)
    return rank[inverse.reshape(-1)], offsets.astype(np.int32)


def levenshtein(a_words: Sequence[str], b_words: Optional[Sequence[str]] = None) -> torch.Tensor:
    """uint8 [A, B] device matrix of unit-cost Levenshtein distances (polyleven.levenshtein on str) between every
    word of a_words and every word of b_words (tip_levenshtein).  b_words None: the square matrix of a_words, each
    unordered pair computed once and mirrored.  Words longer than LEV_MAX_LEN code points raise ValueError before
    anything reaches the device."""
    if b_words is not None:
        check_word_lengths(b_words)          # names the word by its index in b_words
    words = list(a_words) + ([] if b_words is None else list(b_words))
    ids, offsets = encode_words(words)
    dev = require_cuda()
    na = len(a_words)
    nb = na if b_words is None else len(words) - na
    out = torch.empty((na, nb), dtype=torch.uint8, device=dev)
    if na == 0 or nb == 0:
        return out
    lib = _lib.load()
    max_len = int(np.max(np.diff(offsets)))
    ids_d = torch.from_numpy(np.concatenate([ids, np.zeros(1, np.int32)])).to(dev)   # never empty
    off_d = torch.from_numpy(offsets).to(dev)
    if b_words is None:
        a_ids = b_ids = ids_d
        a_off = b_off = off_d
    else:
        a_ids, a_off = ids_d, off_d[:na + 1]
        b_ids, b_off = ids_d[int(offsets[na]):], off_d[na:] - int(offsets[na])
    _lib.check(lib.tip_levenshtein(_p(a_ids), _p(a_off), na, _p(b_ids), _p(b_off), nb, max_len,
                                   int(b_words is None), _p(out), _stream()), "tip_levenshtein")
    return out


# ---- Keras' word tokenizer (tokenizer.cu) ------------------------------------------------------------------------
TOK_HASH_BITS = 64        # hash width of the word tables; narrower only to force collisions in tests


def _pow2_at_least(n: int) -> int:
    return 1 << max(1, int(n - 1).bit_length())


def separator_mask(chars: str) -> Tuple[int, int]:
    """(low, high) 64-bit halves of the 128-bit mask of separator bytes; every char must be ASCII."""
    mask = 0
    for ch in chars:
        if ord(ch) >= 128:
            raise ValueError(f"separator {ch!r} is not ASCII")
        mask |= 1 << ord(ch)
    return mask & (2 ** 64 - 1), mask >> 64


def encode_texts(texts: Sequence[str], lower: bool) -> Tuple[bytes, np.ndarray]:
    """UTF-8 bytes ("surrogatepass": equal str <-> equal bytes) of the texts and their int64 offsets [n + 1].  With
    lower, texts that are not ASCII are lowered here by str.lower(); the device lowers ASCII A-Z, which is
    str.lower() for ASCII text and changes nothing after it."""
    enc = [(t.lower() if lower and not t.isascii() else t).encode("utf-8", "surrogatepass") for t in texts]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum(np.fromiter(map(len, enc), dtype=np.int64, count=len(enc)), out=off[1:])
    if len(enc) and int(np.max(np.diff(off))) >= 2 ** 31:
        raise ValueError("a text has 2^31 bytes or more; word lengths are int32")
    return b"".join(enc), off


class TokWords:
    """The words of one batch of texts on the device (tip_tok_count + tip_tok_emit): the texts' bytes (ASCII
    lowered), word_off [n_texts + 1], and per word (text-major, position-minor) start, length, text and hash."""

    def __init__(self, raw: bytes, off: np.ndarray, sep: Tuple[int, int], lower: bool, hash_bits: int):
        dev = require_cuda()
        lib = _lib.load()
        self.n_texts = len(off) - 1
        self.text = torch.from_numpy(np.frombuffer(bytearray(raw) + b"\0", dtype=np.uint8)).to(dev)   # never empty
        self.text_off = torch.from_numpy(off).to(dev)
        self.word_off = torch.empty(self.n_texts + 1, dtype=torch.int64, device=dev)
        _lib.check(lib.tip_tok_count(_p(self.text), _p(self.text_off), self.n_texts, sep[0], sep[1], int(lower),
                                     _p(self.word_off), _stream()), "tip_tok_count")
        self.n_words = int(self.word_off[-1].item())
        n = max(self.n_words, 1)
        self.start = torch.empty(n, dtype=torch.int64, device=dev)
        self.length = torch.empty(n, dtype=torch.int32, device=dev)
        self.text_id = torch.empty(n, dtype=torch.int32, device=dev)
        self.hash = torch.empty(n, dtype=torch.int64, device=dev)
        _lib.check(lib.tip_tok_emit(_p(self.text), _p(self.text_off), self.n_texts, sep[0], sep[1], _p(self.word_off),
                                    self.n_words, hash_bits, _p(self.start), _p(self.length), _p(self.text_id),
                                    _p(self.hash), _stream()), "tip_tok_emit")


class TokVocab:
    """A tokenizer's vocabulary on the device: its words' bytes (arena, start, length, in word_counts order), their
    Keras indexes, and (built on first use) the open-addressing table that tip_tok_lookup probes."""

    def __init__(self, arena: bytes, start: np.ndarray, length: np.ndarray, index: np.ndarray, hash_bits: int):
        dev = require_cuda()
        self.n = len(start)
        self.hash_bits = hash_bits
        self.arena = torch.from_numpy(np.frombuffer(bytearray(arena) + b"\0", dtype=np.uint8)).to(dev)
        self.start = torch.from_numpy(np.concatenate([start.astype(np.int64), [0]])).to(dev)
        self.length = torch.from_numpy(np.concatenate([length.astype(np.int32), [0]]).astype(np.int32)).to(dev)
        self.index = torch.from_numpy(np.concatenate([index, [0]]).astype(np.int32)).to(dev)
        self.hash = torch.empty(self.n + 1, dtype=torch.int64, device=dev)
        self.keys, self.cap = None, 0

    def table(self, cap: int, first: Optional[torch.Tensor] = None) -> torch.Tensor:
        """keys [cap] of a fresh table holding the vocabulary (tip_tok_vocab_table); first, when given, gets each
        slot's key (the fit's first-occurrence array)."""
        keys = torch.empty(cap, dtype=torch.int64, device=self.hash.device)
        _lib.check(_lib.load().tip_tok_vocab_table(_p(self.arena), _p(self.start), _p(self.length), self.n,
                                                   self.hash_bits, _p(self.hash), _p(keys), _p(first), cap, _stream()),
                   "tip_tok_vocab_table")
        return keys

    def lookup_table(self) -> Tuple[Optional[torch.Tensor], int]:
        if self.keys is None and self.n:
            self.cap = _pow2_at_least(2 * self.n)
            self.keys = self.table(self.cap)
        return self.keys, self.cap


def tok_fit(words: TokWords, vocab: TokVocab) -> np.ndarray:
    """tip_tok_fit of the words against the vocabulary: int64 [5, k] host columns (first-occurrence key, count,
    docs, first byte offset, length) of the k distinct words the batch contains, ordered by first occurrence.  A key
    below vocab.n is that vocabulary entry; a key nv + o is a new word first seen as word o of the batch."""
    dev = words.text.device
    nv, n = vocab.n, words.n_words
    cap, doc_cap = _pow2_at_least(2 * (nv + n)), _pow2_at_least(2 * n)
    first, count, docs = torch.empty((3, cap), dtype=torch.int64, device=dev)
    keys = vocab.table(cap, first)
    doc_keys = torch.empty(doc_cap, dtype=torch.int64, device=dev)
    out = torch.empty((5, nv + n), dtype=torch.int64, device=dev)
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.check(_lib.load().tip_tok_fit(_p(words.text), _p(words.start), _p(words.length), _p(words.text_id),
                                       _p(words.hash), n, _p(vocab.arena), _p(vocab.start), _p(vocab.length),
                                       _p(vocab.hash), nv, _p(keys), _p(first), _p(count), _p(docs), cap, _p(doc_keys),
                                       doc_cap, _p(out), nv + n, _p(n_out), _stream()), "tip_tok_fit")
    cols = out[:, :int(n_out.item())].cpu().numpy()
    return cols[:, np.argsort(cols[0], kind="stable")]


def tok_lookup(words: TokWords, vocab: TokVocab, num_words: int, ragged: bool, maxlen: Optional[int] = None,
               padding: str = "pre", truncating: str = "pre", value: int = 0):
    """tip_tok_lookup: (ragged kept ids int32 or None, kept_off int64 [n_texts + 1], padded int32 [n_texts, maxlen]
    or None) on the device; maxlen None writes no padded rows."""
    dev = words.text.device
    keys, cap = vocab.lookup_table()
    w_id = torch.empty(max(words.n_words, 1), dtype=torch.int32, device=dev)
    kept_off = torch.empty(words.n_texts + 1, dtype=torch.int64, device=dev)
    ids = torch.empty(max(words.n_words, 1), dtype=torch.int32, device=dev) if ragged else None
    padded = None if maxlen is None else torch.empty((words.n_texts, maxlen), dtype=torch.int32, device=dev)
    _lib.check(_lib.load().tip_tok_lookup(_p(words.text), _p(words.start), _p(words.length), _p(words.hash),
                                          words.n_words, _p(vocab.arena), _p(vocab.start), _p(vocab.length),
                                          _p(vocab.hash), _p(vocab.index), vocab.n, _p(keys), cap, num_words,
                                          _p(words.word_off), words.n_texts, _p(w_id), _p(kept_off), _p(ids),
                                          _p(padded), 0 if maxlen is None else maxlen, int(padding == "pre"),
                                          int(truncating == "pre"), value, _stream()), "tip_tok_lookup")
    return ids, kept_off, padded


# ---- IMDB-C's corruptions (corrupt.cu) ---------------------------------------------------------------------------
CORRUPT_CHUNK_BYTES = 1 << 28      # input bytes per chunk; every text is corrupted on its own, so chunking changes nothing
_CP_CLASS = {}                     # code point -> 0 whitespace, 1 word, 2 other, as Python's re classifies it


def _cp_class(cp: int) -> int:
    c = _CP_CLASS.get(cp)
    if c is None:
        ch = chr(cp)
        c = _CP_CLASS[cp] = 0 if re.match(r"\s", ch) else 1 if re.match(r"\w", ch) else 2
    return c


class CorruptTable:
    """One word table of tip_corrupt_words on the device: distinct keys -> lists of strings (cdf: for the common
    words, the flat float64 Generator.choice cdf of every list, in value order).  Strings are stored as UTF-8
    ("surrogatepass"); a lookup compares bytes, so a hash collision never changes a result."""

    def __init__(self, keys: Sequence[str], values: Sequence[Sequence[str]], cdf: Optional[np.ndarray] = None):
        dev = require_cuda()
        n = len(keys)
        enc = [k.encode("utf-8", "surrogatepass") for k in keys]
        enc += [v.encode("utf-8", "surrogatepass") for vals in values for v in vals]
        lens = np.fromiter(map(len, enc), dtype=np.int64, count=len(enc))
        if lens.size and int(lens.max()) >= 2 ** 31:
            raise ValueError("a table string has 2^31 bytes or more")
        off = np.zeros(len(enc), dtype=np.int64)
        np.cumsum(lens[:-1], out=off[1:])
        begin = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.fromiter(map(len, values), dtype=np.int64, count=n), out=begin[1:])

        def up(a, dtype):
            return torch.from_numpy(np.concatenate([np.asarray(a, dtype=dtype), np.zeros(1, dtype)])).to(dev)

        self.n, self.cap = n, _pow2_at_least(2 * n)
        self.arena = torch.from_numpy(np.frombuffer(bytearray(b"".join(enc)) + b"\0", dtype=np.uint8)).to(dev)
        self.key_off, self.key_len = up(off[:n], np.int64), up(lens[:n], np.int32)
        self.val_off, self.val_len = up(off[n:], np.int64), up(lens[n:], np.int32)
        self.val_begin = up(begin, np.int64)
        self.val_cdf = None if cdf is None else up(cdf, np.float64)
        self.key_hash = torch.empty(n + 1, dtype=torch.int64, device=dev)
        self.slots = torch.empty(self.cap, dtype=torch.int32, device=dev)
        self.struct = _lib.CorruptTable(*(t.data_ptr() if t is not None else 0 for t in (
            self.arena, self.key_off, self.key_len, self.key_hash, self.val_begin, self.val_off, self.val_len,
            self.val_cdf, self.slots)), n, self.cap)
        _lib.check(_lib.load().tip_corrupt_table_build(C.addressof(self.struct), _stream()), "tip_corrupt_table_build")


def _class_table(bitmap: torch.Tensor) -> np.ndarray:
    """uint8 [0x110000] classes of ASCII and of the non-ASCII code points the census found (others are never read)."""
    bits = np.unpackbits(bitmap.cpu().numpy().view(np.uint8), bitorder="little")
    cls = np.zeros(bits.size, dtype=np.uint8)
    for cp in list(range(128)) + np.flatnonzero(bits).tolist():
        cls[cp] = _cp_class(cp)
    return cls


def corrupt_texts(encoded: Sequence[bytes], tables: Sequence[CorruptTable], seed: int, severity: float,
                  type_cdf: np.ndarray, chunk_bytes: int = CORRUPT_CHUNK_BYTES,
                  timing: Optional[dict] = None) -> Tuple[list, Optional[int]]:
    """tip_corrupt_* of the strict-UTF-8 texts `encoded` with the (common, bags, thesaurus) tables: (the corrupted
    texts as UTF-8 bytes, None), or (the texts before it, t) when text t is the first with a chosen word whose
    autocorrect has no candidates (the host port raises there).  Texts go in chunks of about chunk_bytes; the result
    does not depend on the chunking.  timing, when given, accumulates "census_ms" (the census and the host's
    classification) and "kernels_ms" (CUDA events around the other launches)."""
    if seed < 0 or not 0.0 <= severity <= 1.0:
        raise ValueError("seed must be >= 0 and severity in [0, 1]")
    cdf = np.ascontiguousarray(type_cdf, dtype=np.float64)
    if cdf.shape != (4,):
        raise ValueError("type_cdf must have 4 entries")
    out, t0 = [], 0
    while t0 < len(encoded):
        t1, size = t0 + 1, len(encoded[t0])
        while t1 < len(encoded) and t1 - t0 < 2 ** 31 - 1 and size + len(encoded[t1]) <= chunk_bytes:
            size += len(encoded[t1])
            t1 += 1
        texts, failed = _corrupt_chunk(encoded[t0:t1], tables, seed, float(severity), cdf, timing)
        out += texts
        if failed is not None:
            return out, t0 + failed
        t0 = t1
    return out, None


def _corrupt_chunk(encoded, tables, seed, severity, cdf, timing):
    dev = require_cuda()
    lib = _lib.load()
    st = _stream()
    n_t = len(encoded)
    off = np.zeros(n_t + 1, dtype=np.int64)
    np.cumsum(np.fromiter(map(len, encoded), dtype=np.int64, count=n_t), out=off[1:])
    if int(np.max(np.diff(off))) >= 2 ** 31:
        raise ValueError("a text has 2^31 bytes or more; word lengths are int32")
    marks = []

    def mark():
        if timing is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append(e)

    c0 = time.perf_counter()
    text = torch.from_numpy(np.frombuffer(bytearray(b"".join(encoded)) + b"\0", dtype=np.uint8)).to(dev)
    text_off = torch.from_numpy(off).to(dev)
    bitmap = torch.empty(_lib.CORRUPT_CP_WORDS, dtype=torch.int32, device=dev)
    _lib.check(lib.tip_corrupt_census(_p(text), int(off[-1]), _p(bitmap), st), "tip_corrupt_census")
    cls = torch.from_numpy(_class_table(bitmap)).to(dev)
    if timing is not None:
        timing["census_ms"] = timing.get("census_ms", 0.0) + 1e3 * (time.perf_counter() - c0)
    mark()
    n_words = torch.empty(n_t, dtype=torch.int64, device=dev)
    _lib.check(lib.tip_corrupt_count(_p(text), _p(text_off), n_t, _p(cls), _p(n_words), st), "tip_corrupt_count")
    mark()
    word_off = np.zeros(n_t + 1, dtype=np.int64)
    np.cumsum(n_words.cpu().numpy(), out=word_off[1:])
    nw = int(word_off[-1])
    word_off_d = torch.from_numpy(word_off).to(dev)
    mark()
    w = max(nw, 1)
    w_start, w_seed, o_off, o_typo, o_pos = torch.empty((5, w), dtype=torch.int64, device=dev)
    w_len, w_cps, w_text, perm, o_len = torch.empty((5, w), dtype=torch.int32, device=dev)
    w_flags, o_src = torch.empty((2, w), dtype=torch.uint8, device=dev)
    err = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.check(lib.tip_corrupt_texts(_p(text), _p(text_off), n_t, _p(cls), _p(word_off_d), seed, severity,
                                     cdf.ctypes.data, _p(w_start), _p(w_len), _p(w_cps), _p(w_text), _p(w_seed),
                                     _p(w_flags), _p(perm), st), "tip_corrupt_texts")
    common, bags, thesaurus = (C.addressof(t.struct) for t in tables)
    _lib.check(lib.tip_corrupt_words(_p(text), _p(w_start), _p(w_len), _p(w_cps), _p(w_seed), _p(w_flags), nw, common,
                                     bags, thesaurus, _p(o_src), _p(o_off), _p(o_len), _p(o_typo), _p(err), st),
               "tip_corrupt_words")
    text_len = torch.empty(n_t, dtype=torch.int64, device=dev)
    _lib.check(lib.tip_corrupt_layout(_p(word_off_d), n_t, _p(o_len), _p(o_typo), _p(o_pos), _p(text_len), st),
               "tip_corrupt_layout")
    mark()
    failed_word = int(err.item())
    if failed_word < nw:
        return [], int(np.searchsorted(word_off, failed_word, side="right")) - 1
    out_off = np.zeros(n_t + 1, dtype=np.int64)
    np.cumsum(text_len.cpu().numpy(), out=out_off[1:])
    out_off_d = torch.from_numpy(out_off).to(dev)
    mark()
    out = torch.empty(max(int(out_off[-1]), 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.tip_corrupt_write(_p(text), _p(w_text), _p(word_off_d), nw, common, bags, thesaurus, _p(o_src),
                                     _p(o_off), _p(o_len), _p(o_typo), _p(o_pos), _p(out_off_d), _p(out), st),
               "tip_corrupt_write")
    mark()
    raw = out[:int(out_off[-1])].cpu().numpy().tobytes()
    if timing is not None:
        # kernel spans only: count, texts / words / layout, write (the gaps hold the host's scans)
        timing["kernels_ms"] = timing.get("kernels_ms", 0.0) + sum(
            marks[i].elapsed_time(marks[i + 1]) for i in (0, 2, 4))
    return [raw[a:b] for a, b in zip(out_off[:-1].tolist(), out_off[1:].tolist())], None


# ---- one training step of the case studies' models (train.cu) ----------------------------------------------------
ADAM_MAX_TENSORS = 256


def adam_table(params: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], m: Sequence[torch.Tensor],
               v: Sequence[torch.Tensor], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """tip_keras_adam's device table of (param, grad, m, v, numel) rows, as uint8 bytes.  Every tensor is a
    contiguous float32 CUDA tensor and each row's four share their shape; ValueError otherwise.  `out`: an existing
    table of the same length to overwrite in place (a captured graph keeps reading it)."""
    n = len(params)
    if not 1 <= n <= ADAM_MAX_TENSORS or not len(grads) == len(m) == len(v) == n:
        raise ValueError(f"tip_keras_adam takes 1..{ADAM_MAX_TENSORS} rows of (param, grad, m, v), got {n}")
    rows = (_lib.AdamTensor * n)()
    for i, ts in enumerate(zip(params, grads, m, v)):
        if any(t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.shape != ts[0].shape
               for t in ts):
            raise ValueError(f"row {i}: param, grad, m and v must be contiguous float32 CUDA tensors of one shape")
        rows[i] = _lib.AdamTensor(*(t.data_ptr() for t in ts), ts[0].numel())
    host = torch.frombuffer(bytearray(rows), dtype=torch.uint8)
    if out is None:
        return host.to(params[0].device)
    out.copy_(host)
    return out


def keras_adam(table: torch.Tensor, n_tensors: int, total_numel: int, state: torch.Tensor, lr: float = 1e-3,
               beta1: float = 0.9, beta2: float = 0.999, epsilon: float = 1e-7) -> None:
    """One Keras Adam step over every tensor of an `adam_table` (tip_keras_adam): state is the device int32 [2]
    (steps taken, 0), advanced by the kernel itself."""
    if state.dtype != torch.int32 or not state.is_cuda or state.numel() != 2:
        raise ValueError("state must be a CUDA int32 tensor of 2 elements")
    lib = _lib.load()
    _lib.check(lib.tip_keras_adam(_p(table), n_tensors, total_numel, _p(state), lr, beta1, beta2, epsilon, _stream()),
               "tip_keras_adam")


def _check_xent_outputs(z, y, loss, dz, correct, m: int) -> None:
    """ValueError unless loss (float32) and correct (int32) hold m elements and every tensor is on z's CUDA device
    (the kernel reads and writes them all through raw pointers)."""
    if loss.numel() < m or correct.numel() < m or loss.dtype != torch.float32 or correct.dtype != torch.int32:
        raise ValueError(f"loss (float32) and correct (int32) need {m} elements")
    if not z.is_cuda or any(t is not None and t.device != z.device for t in (y, loss, dz, correct)):
        raise ValueError(f"z, y, loss, dz and correct must be on one CUDA device, got z on {z.device}")


def softmax_xent(z: torch.Tensor, y: torch.Tensor, loss: torch.Tensor, dz: Optional[torch.Tensor],
                 correct: torch.Tensor) -> None:
    """tip_softmax_xent into preallocated device outputs: loss (float32, 1 element) = the batch mean of the softmax
    cross-entropy of logits z [B, C] against targets y [B, C], dz (None: not written) = (softmax(z) - y) / B, correct
    (int32, 1 element) = rows whose first argmax of z equals that of y."""
    if z.dim() != 2 or y.shape != z.shape or z.dtype != torch.float32 or y.dtype != torch.float32:
        raise ValueError(f"z and y must be float32 [B, C] of one shape, got {tuple(z.shape)}, {tuple(y.shape)}")
    if not (z.is_contiguous() and y.is_contiguous()) or (dz is not None and (dz.shape != z.shape or not dz.is_contiguous())):
        raise ValueError("z, y and dz must be contiguous")
    _check_xent_outputs(z, y, loss, dz, correct, 1)
    lib = _lib.load()
    _lib.check(lib.tip_softmax_xent(_p(z), _p(y), z.shape[0], z.shape[1], _p(loss), _p(dz), _p(correct), _stream()),
               "tip_softmax_xent")


def softmax_xent_seg(z: torch.Tensor, y: torch.Tensor, loss: torch.Tensor, dz: Optional[torch.Tensor],
                     correct: torch.Tensor) -> None:
    """tip_softmax_xent_seg: `softmax_xent` on each of the M segments of logits z [M, B, C] against targets y
    [M, B, C]: loss (float32 [M]), dz (None: not written; else [M, B, C], each segment divided by B) and correct
    (int32 [M]), segment s bit for bit what `softmax_xent(z[s], y[s], ...)` gives."""
    if z.dim() != 3 or y.shape != z.shape or z.dtype != torch.float32 or y.dtype != torch.float32:
        raise ValueError(f"z and y must be float32 [M, B, C] of one shape, got {tuple(z.shape)}, {tuple(y.shape)}")
    if not (z.is_contiguous() and y.is_contiguous()) or (dz is not None and (dz.shape != z.shape or not dz.is_contiguous())):
        raise ValueError("z, y and dz must be contiguous")
    m = z.shape[0]
    _check_xent_outputs(z, y, loss, dz, correct, m)
    lib = _lib.load()
    _lib.check(lib.tip_softmax_xent_seg(_p(z), _p(y), m, z.shape[1], z.shape[2], _p(loss), _p(dz), _p(correct),
                                        _stream()), "tip_softmax_xent_seg")


_GATHER_DTYPES = {torch.float32: (_lib.TIP_F32, torch.float32), torch.float64: (_lib.TIP_F64, torch.float32),
                  torch.int32: (_lib.TIP_I32, torch.int32)}


def check_stack_rows(rows: torch.Tensor, pool_rows: int) -> None:
    """ValueError unless `rows` is a contiguous int64 [M, n] CUDA table of indexes into a pool of `pool_rows` rows
    (one device-to-host read; `stack_gather` relies on it and does not check per step)."""
    if rows.dim() != 2 or rows.dtype != torch.int64 or not rows.is_cuda or not rows.is_contiguous() or rows.numel() == 0:
        raise ValueError(f"rows must be a non-empty contiguous int64 [M, n] CUDA tensor, got {tuple(rows.shape)} "
                         f"{rows.dtype}")
    lo, hi = torch.aminmax(rows)
    lo, hi = int(lo.item()), int(hi.item())
    if lo < 0 or hi >= pool_rows:
        raise ValueError(f"rows index [{lo}, {hi}] outside the pool's {pool_rows} rows")


def stack_gather(pool: torch.Tensor, rows: torch.Tensor, perm: torch.Tensor, start: int, b: int,
                 interleaved: bool = False, out: Optional[torch.Tensor] = None, check: bool = True) -> torch.Tensor:
    """tip_stack_gather: row j < b of model m is `pool[rows[m, perm[m, start + j]]]`, for every model of the rows
    table [M, n] at once (perm [M, n_perm], int64, a permutation of each model's first n_perm rows).

    pool [N, ...] float32, float64 (gathered as float32) or int32 on the device; any other dtype is refused.
    interleaved=False: out [M, b, *row_shape] (model-major); True: a pool of NHWC rows [N, H, W, C] gives out
    [b, H, W, M * C], channel m * C + c of it being model m's channel c.  check=True checks the rows table against
    the pool (`check_stack_rows`, a device-to-host read) and perm against [0, n) (one more); a caller that already
    did passes False, and the values are then not checked."""
    if pool.dtype not in _GATHER_DTYPES:
        raise ValueError(f"tip_stack_gather gathers float32, float64 or int32 pools, not {pool.dtype}")
    if not pool.is_cuda or not pool.is_contiguous() or pool.dim() < 2:
        raise ValueError("pool must be a contiguous CUDA tensor [N, ...]")
    if rows.device != pool.device or perm.device != pool.device:
        raise ValueError(f"rows and perm must be on the pool's device {pool.device}, got {rows.device} and "
                         f"{perm.device}")
    if rows.dim() != 2 or rows.dtype != torch.int64 or not rows.is_contiguous():
        raise ValueError(f"rows must be a contiguous int64 [M, n] tensor, got {tuple(rows.shape)} {rows.dtype}")
    if check:
        check_stack_rows(rows, pool.shape[0])
    if perm.dim() != 2 or perm.dtype != torch.int64 or not perm.is_contiguous() or perm.shape[0] != rows.shape[0]:
        raise ValueError(f"perm must be a contiguous int64 [{rows.shape[0]}, n_perm] tensor, got {tuple(perm.shape)}")
    m, n_rows = rows.shape
    n_perm = perm.shape[1]
    if not (0 <= start and b >= 1 and start + b <= n_perm <= n_rows):
        raise ValueError(f"batch [{start}, {start + b}) outside a permutation of {n_perm} of {n_rows} rows")
    if check:
        lo, hi = torch.stack(torch.aminmax(perm)).tolist()
        if lo < 0 or hi >= n_rows:
            raise ValueError(f"perm index [{lo}, {hi}] outside each model's {n_rows} rows")
    dtype, out_dtype = _GATHER_DTYPES[pool.dtype]
    row_shape = tuple(pool.shape[1:])
    if interleaved:
        if pool.dim() != 4:
            raise ValueError(f"the interleaved layout takes NHWC rows [N, H, W, C], got {tuple(pool.shape)}")
        shape, channels = (b, *row_shape[:-1], m * row_shape[-1]), row_shape[-1]
    else:
        shape, channels = (m, b, *row_shape), 0
    if out is None:
        out = torch.empty(shape, dtype=out_dtype, device=pool.device)
    elif tuple(out.shape) != shape or out.dtype != out_dtype or not out.is_contiguous():
        raise ValueError(f"out must be contiguous {out_dtype} {shape}")
    row_elems = int(np.prod(row_shape))
    _lib.check(_lib.load().tip_stack_gather(_p(pool), dtype, row_elems, _p(rows), n_rows, _p(perm), n_perm, start, b,
                                            m, channels, _p(out), _stream()), "tip_stack_gather")
    return out


MC_MAX_LAYERS = 4         # dense layers of an MC-dropout head
MC_MAX_IN = 8192          # the head's input width (the trunk's)
MC_MAX_WIDTH = 64         # units of every head layer
MC_ACTIVATIONS = {None: _lib.MC_LINEAR, "linear": _lib.MC_LINEAR, "relu": _lib.MC_RELU, "softmax": _lib.MC_SOFTMAX}


def _mc_table(layers, width: int, dev, models: Optional[int] = None):
    """(tip_mc_layer table, the last layer's width) of engine.mc_head's `layers` on `width` inputs; models = M: each
    kernel [M, in, out] and bias [M, out] (mc_head_stack).  ValueError for anything else."""
    if not 1 <= len(layers) <= MC_MAX_LAYERS:
        raise ValueError(f"an MC-dropout head has 1..{MC_MAX_LAYERS} dense layers, got {len(layers)}")
    if not 1 <= width <= MC_MAX_IN:
        raise ValueError(f"the head's input width must be 1..{MC_MAX_IN}, got {width}")
    lead = () if models is None else (models,)
    table = (_lib.McLayer * len(layers))()
    for i, (kernel, bias, p, act) in enumerate(layers):
        if act not in MC_ACTIVATIONS or (act == "softmax" and i != len(layers) - 1):
            raise ValueError(f"layer {i}: activation {act!r} (linear, relu, or softmax on the last layer)")
        for name, t, dim in (("kernel", kernel, 2 + len(lead)), ("bias", bias, 1 + len(lead))):
            if (not isinstance(t, torch.Tensor) or t.dim() != dim or t.dtype != torch.float32 or t.device != dev
                    or not t.is_contiguous()):
                raise ValueError(f"layer {i}: {name} must be a contiguous {dim}-D float32 tensor on {dev}")
        out = kernel.shape[-1]
        if (tuple(kernel.shape[:-1]) != (*lead, width) or not 1 <= out <= MC_MAX_WIDTH
                or tuple(bias.shape) != (*lead, out)):
            raise ValueError(f"layer {i}: kernel {tuple(kernel.shape)} / bias {tuple(bias.shape)} do not take {width} "
                             f"inputs to 1..{MC_MAX_WIDTH} units" + (f" for {models} models" if lead else ""))
        p = float(p)
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"layer {i}: dropout rate {p} outside [0, 1]")
        table[i] = _lib.McLayer(kernel.data_ptr(), bias.data_ptr(), p, width, out, MC_ACTIVATIONS[act], 0)
        width = out
    return table, width


def mc_head(h: torch.Tensor, layers, seed: int, samples: int, row0: int = 0, sample0: int = 0,
            out: Optional[torch.Tensor] = None, preact: bool = False) -> torch.Tensor:
    """tip_mc_head: `samples` MC-dropout samples of a dense head for every row of the trunk activations h
    [rows, D] (float32 on the current CUDA device, unit column stride, any row stride).  layers: 1..4 tuples
    (kernel [in, out], bias [out], p, activation), kernel and bias contiguous float32 on h's device, p the dropout
    rate on the layer's input (0: none), activation None / "linear" / "relu" / "softmax" (softmax only last);
    D <= 8192, every out <= 64.  Row i of h is global row row0 + i and sample s global sample sample0 + s: the masks
    depend on (seed, layer, global row, global sample, unit) only (include/b200tip.h).  Returns out [rows, samples,
    C] float32: the last layer's output, or its pre-activation (preact=True).  Raises ValueError before any launch
    for anything else."""
    dev = require_cuda()
    if not isinstance(h, torch.Tensor) or h.dim() != 2 or h.dtype != torch.float32 or h.device != dev:
        raise ValueError(f"h must be a 2-D float32 tensor on {dev}, got "
                         f"{tuple(h.shape) if isinstance(h, torch.Tensor) else type(h).__name__}")
    if h.shape[0] > 0 and h.shape[1] > 1 and h.stride(1) != 1:
        raise ValueError("h must have a unit column stride")
    if not 1 <= len(layers) <= MC_MAX_LAYERS:
        raise ValueError(f"an MC-dropout head has 1..{MC_MAX_LAYERS} dense layers, got {len(layers)}")
    if samples < 1 or row0 < 0 or sample0 < 0:
        raise ValueError(f"samples >= 1, row0 >= 0 and sample0 >= 0, got {samples}, {row0}, {sample0}")
    table, width = _mc_table(layers, h.shape[1], dev)
    rows = h.shape[0]
    shape = (rows, samples, width)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=dev)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != dev or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float32 {shape} tensor on {dev}")
    ld = h.stride(0) if rows > 1 else h.shape[1]
    _lib.check(_lib.load().tip_mc_head(_p(h), rows, ld, row0, sample0, samples, table, len(layers),
                                       int(seed) & 0xFFFFFFFFFFFFFFFF, _lib.MC_PREACT if preact else _lib.MC_OUTPUT,
                                       _p(out), _stream()), "tip_mc_head")
    return out


def mc_head_stack(h: torch.Tensor, layers, seeds, samples: int, row0: int = 0, sample0: int = 0,
                  out: Optional[torch.Tensor] = None, preact: bool = False) -> torch.Tensor:
    """tip_mc_head_stack: `mc_head` for the M heads of one shape of a stack, in one launch per 256 models.  h
    [M, rows, D] (float32 on the current CUDA device, unit column stride, any row and model stride: a model stride
    of 0, as `expand` gives, feeds every model the same rows); layers: 1..4 tuples (kernel [M, in, out], bias [M,
    out], p, activation) as `mc_head` takes them with a leading model axis; seeds: M ints.  Returns out [M, rows,
    samples, C] float32, whose slice m is bit for bit `mc_head(h[m], model m's layers, seeds[m], ...)`.  Raises
    ValueError before any launch for anything else."""
    dev = require_cuda()
    if not isinstance(h, torch.Tensor) or h.dim() != 3 or h.dtype != torch.float32 or h.device != dev:
        raise ValueError(f"h must be a 3-D float32 tensor [M, rows, D] on {dev}, got "
                         f"{tuple(h.shape) if isinstance(h, torch.Tensor) else type(h).__name__}")
    models, rows, d = h.shape
    if models * rows > 0 and d > 1 and h.stride(2) != 1:
        raise ValueError("h must have a unit column stride")
    if min(h.stride()) < 0:
        raise ValueError("h must have non-negative strides")
    seeds = [int(s) for s in seeds]
    if len(seeds) != models:
        raise ValueError(f"{len(seeds)} seeds for {models} models")
    if samples < 1 or row0 < 0 or sample0 < 0:
        raise ValueError(f"samples >= 1, row0 >= 0 and sample0 >= 0, got {samples}, {row0}, {sample0}")
    table, width = _mc_table(layers, d, dev, models)
    shape = (models, rows, samples, width)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=dev)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != dev or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float32 {shape} tensor on {dev}")
    ld = h.stride(1) if rows > 1 else d
    ldm = h.stride(0) if models > 1 else 0
    seed_table = (C.c_uint64 * max(models, 1))(*[s & 0xFFFFFFFFFFFFFFFF for s in seeds])
    _lib.check(_lib.load().tip_mc_head_stack(_p(h), models, rows, ld, ldm, row0, sample0, samples, table, len(layers),
                                             seed_table, _lib.MC_PREACT if preact else _lib.MC_OUTPUT, _p(out),
                                             _stream()), "tip_mc_head_stack")
    return out
