"""CTM / CAM orderings — reference: src/core/prioritizers.py:7-59 (SURVEY.md §8 f1).

`ctm` / `cam` keep the reference's signatures; `cam`'s greedy loop runs on the GPU over the bit-packed
profile (`cam_from_bits`, one persistent cooperative kernel), which is also the entry point for profiles that
never left HBM (`NAC/NBC/SNAC/TKNC.packed`); `cam_from_bits_stack` orders the profiles of a model stack's M models
in one such kernel.  `cam_from_buckets` is the same ordering for k-multisection profiles given in their compact form
(the bucket ids of `KMNC.buckets`): the greedy loop runs on the GPU (libb200tip `tip_cam_buckets`)
without ever building the N x D x k array, which is 41 GB at k = 1000.  `cam_from_surprise` is the ordering for
surprise-coverage profiles (`SurpriseCoverageMapper`): one pass over the scores (libb200tip `tip_sc_cam`)."""
import itertools
from typing import Generator, List, Sequence

import numpy as np


def ctm(scores: np.ndarray) -> Generator[int, None, None]:
    """Coverage-total method: indexes by decreasing score (`np.argsort(-scores)`)."""
    assert len(scores.shape) == 1
    yield from np.argsort(-scores)


LAST_GREEDY_PICKS = 0      # greedy rounds of the most recent CAM call (bench / diagnostics)
LAST_GREEDY_MS = 0.0       # device time of its greedy loop (CUDA events around the launches)


def _tail_by_score(scores: np.ndarray, greedy: np.ndarray):
    """prioritizers.py:47-59: the samples the greedy loop did not yield, by `np.argsort(-scores)` — NumPy's
    own (unstable) sort on the host, so ties fall exactly as in the reference."""
    n = scores.shape[0]
    if n == 0:
        return
    taken = np.zeros(n, dtype=bool)
    taken[greedy] = True
    floor = np.min(scores) - 1
    scores[taken] = floor - 1
    for i in np.argsort(-scores):
        if scores[i] < floor:
            break
        yield int(i)


def _greedy_bits(bits, rounds_per_launch: int, stack: bool):
    """The greedy picks of M profiles, bits [M, N, words] int32 CUDA tensor with N, words >= 1, and the device time
    of the loop in ms (CUDA events around the launches).  The loop is libb200tip `tip_cam_bits_stack`, or
    `tip_cam_bits` when not `stack` (M = 1), launched until no model is still live (not done and fewer than N
    picks), `rounds_per_launch` rounds per launch.  Returns (M int64 pick arrays, ms)."""
    import torch

    from .. import _lib
    from .. import engine as E

    lib = _lib.load()
    models, n, words = (int(s) for s in bits.shape)
    entry, dims = ("tip_cam_bits_stack", (models, n, words)) if stack else ("tip_cam_bits", (n, words))
    dev = bits.device
    bits = bits.contiguous()
    gain = torch.empty((models, n), dtype=torch.int32, device=dev)
    covered = torch.zeros((models, 2 * words), dtype=torch.int32, device=dev)
    cand = torch.zeros(4 * _lib.CAM_MAX_BLOCKS, dtype=torch.int32, device=dev)
    order = torch.zeros((models, n), dtype=torch.int32, device=dev)
    state = torch.zeros((models, 4), dtype=torch.int32, device=dev)
    rounds = max(2, int(rounds_per_launch) & ~1)              # even: the covered sets are double-buffered by parity
    first = 1
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    while True:
        _lib.check(getattr(lib, entry)(E._p(bits), *dims, E._p(gain), E._p(covered), E._p(cand), E._p(order),
                                       E._p(state), rounds, first, E._stream()), entry)
        first = 0
        ev1.record()
        st = state.cpu().numpy()
        if not np.any((st[:, 1] == 0) & (st[:, 0] < n)):
            break
    picked = order[:, :int(st[:, 0].max())].cpu().numpy()
    return [picked[m, :st[m, 0]].astype(np.int64) for m in range(models)], float(ev0.elapsed_time(ev1))


def cam_from_bits(scores: np.ndarray, bits, rounds_per_launch: int = 4096) -> Generator[int, None, None]:
    """`cam(scores, profiles)` for a boolean profile given bit-packed in HBM: bits [N, words] int32 CUDA
    tensor (any consistent packing — `NAC/NBC/SNAC/TKNC.packed()` or `pack_profiles`).  The greedy loop
    (prioritizers.py:24-45) is ONE persistent cooperative kernel (libb200tip `tip_cam_bits`): per round an
    arg-max of the gains, new = profile[pick] & ~covered, gain -= popcount(profile & new)."""
    scores = np.asarray(scores).copy()
    assert scores.ndim == 1
    n, words = int(bits.shape[0]), int(bits.shape[1]) if bits.ndim == 2 else 0
    assert scores.shape[0] == n, "one score per sample"
    greedy = np.zeros(0, dtype=np.int64)
    if n > 0 and words > 0:
        global LAST_GREEDY_MS
        (greedy,), LAST_GREEDY_MS = _greedy_bits(bits[None], rounds_per_launch, stack=False)
    global LAST_GREEDY_PICKS
    LAST_GREEDY_PICKS = int(greedy.shape[0])
    yield from (int(i) for i in greedy)
    yield from _tail_by_score(scores, greedy)


def cam_from_bits_stack(scores: Sequence[np.ndarray], bits, rounds_per_launch: int = 4096) -> List[np.ndarray]:
    """`cam_from_bits` for the profiles of M models at once (a model stack's): bits [M, N, words] int32 CUDA tensor,
    scores M vectors of N.  The M greedy loops run in one persistent cooperative kernel (libb200tip
    `tip_cam_bits_stack`), one grid barrier per round for all of them; each model's remaining samples then follow
    by its scores on the host (`_tail_by_score`).  Returns, per model m, the int64 order
    `list(cam_from_bits(scores[m], bits[m]))` gives."""
    scores = [np.asarray(s).copy() for s in scores]
    assert bits.ndim == 3, "bits [M, N, words]"
    models, n, words = (int(s) for s in bits.shape)
    assert len(scores) == models and all(s.ndim == 1 and s.shape[0] == n for s in scores), "M vectors of N scores"
    greedy = [np.zeros(0, dtype=np.int64)] * models
    if models > 0 and n > 0 and words > 0:
        greedy, _ = _greedy_bits(bits, rounds_per_launch, stack=True)
    return [np.fromiter(itertools.chain(g, _tail_by_score(s, g)), dtype=np.int64) for s, g in zip(scores, greedy)]


def pack_profiles(profiles):
    """Dense boolean profiles [N, ...] (NumPy or torch, host or device) -> bit-packed [N, ceil(F/32)] int32
    CUDA tensor (libb200tip `tip_pack_bool`)."""
    import torch

    from .. import _lib
    from .. import engine as E

    dev = E.require_cuda()
    if isinstance(profiles, torch.Tensor):
        p = profiles.reshape(profiles.shape[0], -1).to(dev)
        p = (p != 0).to(torch.uint8).contiguous() if p.dtype != torch.bool else p.contiguous()
    else:
        flat = np.ascontiguousarray(np.asarray(profiles).reshape((profiles.shape[0], -1)))
        p = torch.from_numpy(flat.view(np.uint8) if flat.dtype == np.bool_ else (flat != 0).view(np.uint8)).to(dev)
    n, f = int(p.shape[0]), int(p.shape[1])
    words = (f + 31) // 32
    bits = torch.empty((n, max(words, 0)), dtype=torch.int32, device=dev)
    if n and f:
        _lib.check(_lib.load().tip_pack_bool(E._p(p), n, f, E._p(bits), E._stream()), "tip_pack_bool")
    return bits


def cam(scores: np.ndarray, profiles: np.ndarray) -> Generator[int, None, None]:
    """Coverage-additional method (prioritizers.py:16-59): greedily pick the sample covering the most
    still-uncovered profile entries (first index on ties, like np.argmax); once nothing new can be
    covered, the remaining samples follow by decreasing score.  Same signature as the reference (dense
    boolean profiles of any shape [N, ...]); the profile is bit-packed on the GPU and the greedy loop runs
    there (`cam_from_bits`)."""
    scores = np.asarray(scores)
    assert len(scores.shape) == 1
    yield from cam_from_bits(scores, pack_profiles(profiles))


def cam_from_buckets(scores: np.ndarray, bucket, sections: int) -> Generator[int, None, None]:
    """`cam(scores, profiles)` for the one-hot-per-neuron profile whose compact form is
    bucket[n, d] in {-1, 0..sections-1} (NumPy array or torch CUDA tensor, int16 / int32, e.g. from
    `KMNC.buckets(..., device_out=True)`).  Yields exactly the indexes the reference's generator yields
    on the dense profile (prioritizers.py:16-59): greedy picks from the GPU, then the remaining samples
    by `np.argsort(-scores)` on the host (NumPy's own sort, so ties fall as in the reference)."""
    import torch

    from .. import _lib
    from .. import engine as E

    scores = np.asarray(scores).copy()
    assert scores.ndim == 1
    dev = E.require_cuda()
    lib = _lib.load()
    b = bucket if isinstance(bucket, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(bucket))
    if b.dtype not in (torch.int16, torch.int32):
        b = b.to(torch.int32)
    b = b.to(dev).contiguous()
    n, d = b.shape
    assert scores.shape[0] == n, "one score per sample"
    if n > 0 and d > 0:
        gain = ((b >= 0) & (b < int(sections))).sum(dim=1, dtype=torch.int32).contiguous()   # valid cells per sample
        covered = torch.zeros((d * int(sections) + 31) // 32, dtype=torch.int32, device=dev)
        newlist = torch.empty(2 * d, dtype=torch.int32, device=dev)
        order = torch.zeros(n, dtype=torch.int32, device=dev)
        state = torch.zeros(4, dtype=torch.int32, device=dev)
        bdt = _lib.TIP_I16 if b.dtype == torch.int16 else _lib.TIP_I32
        picks, done, rounds = 0, False, 64
        while not done and picks < n:
            _lib.check(lib.tip_cam_buckets(E._p(b), bdt, n, d, int(sections), E._p(gain), E._p(covered), E._p(newlist),
                                           E._p(order), E._p(state), min(rounds, n - picks), E._stream()),
                       "tip_cam_buckets")
            st = state.cpu().numpy()
            picks, done = int(st[0]), bool(st[1])
            rounds = min(4 * rounds, 1024)       # a sync every few hundred rounds is noise
        greedy = order[:picks].cpu().numpy().astype(np.int64)
    else:
        greedy = np.zeros(0, dtype=np.int64)
    global LAST_GREEDY_PICKS
    LAST_GREEDY_PICKS = int(greedy.shape[0])
    yield from (int(i) for i in greedy)
    yield from _tail_by_score(scores, greedy)


def thresholds_one_hot(thresholds: np.ndarray) -> bool:
    """True when the bucket edges are NaN-free and non-decreasing, so that the buckets [t[b], t[b+1]) are disjoint
    and every row of `SurpriseCoverageMapper.get_coverage_profile` holds at most one True.  np.linspace breaks this
    for a negative, NaN or +inf upper bound (+inf is what np.max picks up from LSA scores whose density underflowed)."""
    t = np.asarray(thresholds, dtype=np.float64)
    return not np.isnan(t).any() and bool(np.all(t[1:] >= t[:-1]))


def cam_from_surprise(scores, mapper) -> Generator[int, None, None]:
    """`cam(scores, mapper.get_coverage_profile(scores))` for a `SurpriseCoverageMapper` (handler_surprise.py:101-115),
    without the N x sections profile.  scores: float32 or float64, NumPy or a CUDA tensor.

    When the mapper's thresholds pass `thresholds_one_hot`, the profile is one-hot, and the reference's greedy loop
    picks the first sample of every non-empty bucket in ascending sample order: one pass over the scores on the GPU
    (libb200tip `tip_sc_cam`) finds them.  Otherwise the dense profile is built with the mapper's own expression and
    ordered by `cam`.  The rest follows by `np.argsort(-scores)` on the host in the scores' own dtype, so ties fall
    as in the reference.  At most `_lib.SC_CAM_MAX_SECTIONS` sections (ValueError before any launch)."""
    import torch

    from .. import _lib
    from .. import engine as E

    thresholds = np.asarray(mapper.thresholds, dtype=np.float64)
    sections = thresholds.shape[0] - 1
    if not 1 <= sections <= _lib.SC_CAM_MAX_SECTIONS:
        raise ValueError(f"cam_from_surprise takes 1 to {_lib.SC_CAM_MAX_SECTIONS} sections, got {sections}")
    on_device = isinstance(scores, torch.Tensor)
    host = scores.detach().cpu().numpy() if on_device else np.asarray(scores)
    assert host.ndim == 1
    dtype = E.tip_dtype(host.dtype)
    if not thresholds_one_hot(thresholds):
        yield from cam(host, mapper.get_coverage_profile(host))
        return
    n = host.shape[0]
    greedy = np.zeros(0, dtype=np.int64)
    if n > 0:
        dev = E.require_cuda()
        values = scores.detach().to(dev).contiguous() if on_device else torch.from_numpy(np.ascontiguousarray(host)).to(dev)
        t = torch.from_numpy(thresholds).to(dev)
        first = torch.empty(sections, dtype=torch.int32, device=dev)
        out = torch.empty(sections + 1, dtype=torch.int32, device=dev)          # [count, order...]: one download
        _lib.check(_lib.load().tip_sc_cam(E._p(values), dtype, n, E._p(t), sections, E._p(first), E._p(out[1:]),
                                          E._p(out), E._stream()), "tip_sc_cam")
        res = out.cpu().numpy()
        greedy = res[1:1 + int(res[0])].astype(np.int64)
    global LAST_GREEDY_PICKS
    LAST_GREEDY_PICKS = int(greedy.shape[0])
    yield from (int(i) for i in greedy)
    yield from _tail_by_score(host.copy(), greedy)
