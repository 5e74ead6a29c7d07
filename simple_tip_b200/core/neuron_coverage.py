"""Neuron-coverage criteria behind the reference's `src.core.neuron_coverage` API.

KMNC (neuron_coverage.py:65-94 of the reference) is scored by libb200tip.so: one streaming
pass computes, per (sample, neuron), the section index i with
`thresh[i] <= a < thresh[i+1]` (thresholds `min + jumps*i` re-evaluated on the fly with NumPy's
rounding) and the per-sample count, i.e. the compact form of the reference's dense
N x D x sections boolean profile.  `KMNC.__call__` expands it to the dense profile only because
the reference API returns one (consumers: `cam`, handler_coverage.py:122-124); `buckets()` is the
compact entry point for large `sections`, `packed()` the same sections bit-packed in HBM (one plane per section).  NAC / NBC / SNAC / TKNC (neuron_coverage.py:52-62,97-173)
run on the GPU as well (csrc/coverage.cu): the boundaries are the reference's NumPy expressions, the
comparisons happen in NumPy's promoted dtype, so scores and profiles are bit-identical; every class
also offers `packed(...)`, the same profile bit-packed in HBM for `prioritizers.cam_from_bits`.
"""
from __future__ import annotations

import abc
from typing import List, Tuple

import numpy as np


def sum_score(profiles: np.ndarray) -> np.ndarray:
    """Count of covered profile entries per sample, in the narrowest of int16/32/64 that can
    hold the maximum (neuron_coverage.py:8-22)."""
    assert profiles.dtype == np.bool_
    return np.sum(profiles.reshape((profiles.shape[0], -1)), axis=1, dtype=_score_dtype(np.prod(profiles[0].shape)))


def _score_dtype(max_value: int):
    if max_value <= np.iinfo(np.int16).max:
        return np.int16
    if max_value <= np.iinfo(np.int32).max:
        return np.int32
    return np.int64


def flatten_layers(layers: List[np.ndarray]) -> np.ndarray:
    return np.concatenate([np.reshape(l, (l.shape[0], -1)) for l in layers], axis=1)


class CoverageMethod(abc.ABC):
    def __init__(self):
        pass

    @abc.abstractmethod
    def __call__(self, activations: List[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        ...


def _device_activations(activations):
    """Activations (NumPy array / list of layers / torch CUDA tensors) as one contiguous [N, D] matrix in
    HBM, its NumPy dtype there, and the NumPy dtype the activations came in.  float32 / float64 are kept;
    everything else is widened exactly (float16, bool and small integers to float32, wider integers to
    float64).  The comparison dtype is NumPy's promotion of the ORIGINAL dtype with the boundaries (the
    caller's job).  A torch bfloat16 tensor has no NumPy dtype: it counts as float32."""
    import torch

    from .. import engine as E

    dev = E.require_cuda()
    dev_act = E.device_matrix(activations)
    if dev_act is not None:
        orig = np.dtype(np.float32) if dev_act.dtype == torch.bfloat16 else torch.empty(0, dtype=dev_act.dtype).numpy().dtype
        wide = np.result_type(orig, np.float32)
        if wide not in (np.float32, np.float64):
            raise TypeError(f"unsupported activation dtype {dev_act.dtype}")
        act = dev_act if dev_act.dtype in (torch.float32, torch.float64) else dev_act.to(
            torch.float64 if wide == np.float64 else torch.float32)
        return act.contiguous(), E.NP_DTYPE[act.dtype], orig
    if isinstance(activations, np.ndarray):
        act = activations.reshape((activations.shape[0], -1))
    elif len(activations) == 1:
        act = np.reshape(activations[0], (activations[0].shape[0], -1))
    else:
        act = flatten_layers(activations)
    orig = act.dtype
    if act.dtype not in (np.float32, np.float64):
        act = act.astype(np.result_type(act.dtype, np.float32))
        if act.dtype not in (np.float32, np.float64):
            raise TypeError(f"unsupported activation dtype {act.dtype}")
    return E.to_device(act, dev), act.dtype, orig


class _ThresholdCoverage(CoverageMethod):
    """Shared launch path of NAC / SNAC / NBC (tip_cover_threshold)."""

    _mode = None
    _planes = 1

    def _bounds(self):
        """(lo, hi, scalar threshold): NumPy arrays / None as the criterion defines them"""
        raise NotImplementedError

    def _run(self, activations, want_profile: bool, want_bits: bool):
        import torch

        from .. import _lib
        from .. import engine as E

        lib = _lib.load()
        act, act_dt, orig_dt = _device_activations(activations)
        dev = act.device
        n, d = act.shape
        lo, hi, thr = self._bounds()
        if hi is not None:
            assert d == hi.shape[0], "activation width does not match the boundary statistics"
            stat_dt = np.result_type(hi.dtype, np.float32) if hi.dtype.kind != "f" else hi.dtype
            if stat_dt not in (np.float32, np.float64):
                stat_dt = np.dtype(np.float64)
            key = ("bounds", str(stat_dt), str(dev))
            if getattr(self, "_dev_key", None) != key:
                self._dev_hi = E.to_device(np.ascontiguousarray(hi, dtype=stat_dt), dev)
                self._dev_lo = None if lo is None else E.to_device(np.ascontiguousarray(lo, dtype=stat_dt), dev)
                self._dev_key = key
            lo_dev, hi_dev = self._dev_lo, self._dev_hi
            thr_val = 0.0
        else:
            # NAC: `activations > threshold` with a Python / NumPy scalar: NumPy compares in the promotion of the
            # activations' own dtype with the threshold (float16 stays float16, int16 against a Python float is
            # float64).  The threshold is rounded to that dtype; the kernel then compares in float64 when it is
            # float64 or an integer type, else in float32, which is exact for float16 values.
            cmp_dt = np.result_type(orig_dt, thr)
            stat_dt = np.dtype(np.float32) if cmp_dt in (np.float16, np.float32) else np.dtype(np.float64)
            lo_dev = hi_dev = None
            thr_val = float(np.asarray(thr).astype(cmp_dt)) if cmp_dt.kind == "f" else float(thr)
        profile = torch.empty((n, d) if self._planes == 1 else (n, d, 2), dtype=torch.bool, device=dev) if want_profile else None
        words = int(lib.tip_cover_packed_words(d))
        bits = torch.empty((n, self._planes * words), dtype=torch.int32, device=dev) if want_bits else None
        score = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(lib.tip_cover_threshold(E._p(act), E.tip_dtype(act_dt), n, d, E._p(lo_dev), E._p(hi_dev),
                                           E.tip_dtype(stat_dt), thr_val, self._mode, E._p(profile), E._p(bits),
                                           E._p(score), E._stream()), "tip_cover_threshold")
        return score, profile, bits, d

    def __call__(self, activations: List[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        score, profile, _, d = self._run(activations, True, False)
        return score.cpu().numpy().astype(_score_dtype(d * self._planes)), profile.cpu().numpy()

    def packed(self, activations):
        """(scores int32 [N], profile bit-packed [N, words] int32) as CUDA tensors — nothing leaves HBM; feed
        to `prioritizers.cam_from_bits`."""
        score, _, bits, _ = self._run(activations, False, True)
        return score, bits


class NAC(_ThresholdCoverage):
    """Neuron activation coverage: a > threshold (neuron_coverage.py:52-62)."""

    _mode = 0

    def __init__(self, cov_threshold: float):
        super().__init__()
        self.cov_threshold = cov_threshold

    def _bounds(self):
        return None, None, self.cov_threshold


class KMNC(CoverageMethod):
    """k-multisection neuron coverage on the GPU."""

    def __init__(self, mins: List[np.ndarray], maxs: List[np.ndarray], sections: int):
        super().__init__()
        self.sections = sections
        lo = np.concatenate([np.asarray(l).flatten() for l in mins])
        hi = np.concatenate([np.asarray(l).flatten() for l in maxs])
        jumps = (hi - lo) / sections                       # neuron_coverage.py:76 (same NumPy expression)
        self._lo, self._jumps = lo + jumps * 0, jumps       # lo promoted to the threshold dtype
        self._dev_stats = None

    @property
    def thresh(self) -> List[np.ndarray]:
        """The reference's threshold list (neuron_coverage.py:79), built on demand."""
        lo = self._lo
        return [lo + self._jumps * i for i in range(self.sections + 1)]

    def _prepare(self, activations):
        """(activations as one [N, D] matrix — a contiguous CUDA tensor, or a NumPy array still on the host —, whether
        it came from the device, its NumPy dtype, the statistics' dtype)"""
        import torch

        from .. import engine as E

        dev_act = E.device_matrix(activations)
        if dev_act is not None:
            act = dev_act if dev_act.dtype in (torch.float32, torch.float64) else dev_act.to(torch.float32)
            act = act.contiguous()
        elif isinstance(activations, np.ndarray):   # (explicit widths: a -1 cannot be resolved for 0 samples)
            act = activations.reshape((activations.shape[0], int(np.prod(activations.shape[1:]))))
        elif len(activations) == 1:          # one layer: no concatenation copy (keeps a pinned buffer pinned)
            act = np.reshape(activations[0], (activations[0].shape[0], int(np.prod(activations[0].shape[1:]))))
        else:
            act = flatten_layers(activations)
        stat_dt = self._jumps.dtype
        if stat_dt not in (np.float32, np.float64):
            raise TypeError(f"KMNC statistics must be float32/float64 after NumPy promotion, got {stat_dt}")
        if dev_act is None and act.dtype not in (np.float32, np.float64):
            act = act.astype(np.result_type(act.dtype, stat_dt))
            if act.dtype not in (np.float32, np.float64):
                raise TypeError(f"unsupported activation dtype {act.dtype}")
        act_np_dtype = E.NP_DTYPE[act.dtype] if dev_act is not None else act.dtype
        assert act.shape[1] == self._lo.shape[0], "activation width does not match the min/max statistics"
        return act, dev_act is not None, act_np_dtype, stat_dt

    def _device_stats(self, dev):
        from .. import engine as E

        if self._dev_stats is None:
            self._dev_stats = (E.to_device(self._lo.astype(self._jumps.dtype), dev), E.to_device(self._jumps, dev))
        return self._dev_stats

    def buckets(self, activations, device_out: bool = False):
        """(scores [N] in the reference's score dtype — int32 CUDA tensor with device_out —, bucket ids [N, D] int16/int32;
        -1 = no section covered).
        Activations may be NumPy arrays or device-resident torch tensors (one or a list);
        device_out=True returns the two results as CUDA tensors (no D2H of the N x D bucket ids)."""
        import torch

        from .. import _lib
        from .. import engine as E

        act, on_device, act_np_dtype, stat_dt = self._prepare(activations)
        dev = E.require_cuda()
        lib = _lib.load()
        n, d = act.shape
        lo_dev, jump_dev = self._device_stats(dev)
        small = self.sections <= np.iinfo(np.int16).max
        bdt, btag = (torch.int16, _lib.TIP_I16) if small else (torch.int32, _lib.TIP_I32)

        def launch(a_chunk, bucket_chunk, score_chunk):
            _lib.check(lib.tip_kmnc(E._p(a_chunk), E.tip_dtype(act_np_dtype), a_chunk.shape[0], d, E._p(lo_dev), E._p(jump_dev),
                                    E.tip_dtype(stat_dt), self.sections, E._p(bucket_chunk), btag, E._p(score_chunk),
                                    E._stream()), "tip_kmnc")

        if device_out or on_device or n * d * act.dtype.itemsize < self.PIPELINE_BYTES:
            a_dev = E.to_device(act, dev)
            bucket = torch.empty((n, d), dtype=bdt, device=dev)
            score = torch.empty(n, dtype=torch.int32, device=dev)
            launch(a_dev, bucket, score)
            if device_out:
                return score, bucket
            hb, hs = self._host_buffers(n, d, bdt)
            hb.copy_(bucket, non_blocking=True)
            hs.copy_(score, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            # scores in the dtype the reference's sum_score picks (int16 / int32 / int64 by D * sections): np.argsort's tie
            # order — and with it ctm / the tail of cam — depends on the dtype
            return hs.numpy().astype(_score_dtype(d * self.sections)), hb.numpy().copy()
        # Large host batches: PCIe is the bound (C4: 164 MB up, 82 MB down), so rows go through in chunks with the
        # upload of chunk i+1, the kernel of chunk i and the download of chunk i-1 in flight together (full duplex).
        hb, hs = self._host_buffers(n, d, bdt)
        src = torch.from_numpy(np.ascontiguousarray(act))
        main = torch.cuda.current_stream()
        up, down = self._side_streams(dev)
        rows = max(256, -(-n // self.PIPELINE_CHUNKS))
        # device staging recycled per shape: side-stream use would otherwise keep the caching allocator from reusing
        # the blocks (fresh cudaMalloc of 250 MB per call)
        dkey = (n, d, src.dtype, bdt)
        if getattr(self, "_dev_key2", None) != dkey:
            self._dev_bufs = (torch.empty((n, d), dtype=src.dtype, device=dev), torch.empty((n, d), dtype=bdt, device=dev),
                              torch.empty(n, dtype=torch.int32, device=dev))
            self._dev_key2 = dkey
        a_dev, bucket, score = self._dev_bufs
        up.wait_stream(main)
        down.wait_stream(main)
        landed = []
        for r0 in range(0, n, rows):
            r1 = min(n, r0 + rows)
            with torch.cuda.stream(up):
                a_dev[r0:r1].copy_(src[r0:r1], non_blocking=True)
                ready = torch.cuda.Event()
                ready.record()
            main.wait_event(ready)
            launch(a_dev[r0:r1], bucket[r0:r1], score[r0:r1])
            done = torch.cuda.Event()
            done.record()
            down.wait_event(done)
            with torch.cuda.stream(down):
                hb[r0:r1].copy_(bucket[r0:r1], non_blocking=True)
                hs[r0:r1].copy_(score[r0:r1], non_blocking=True)
                here = torch.cuda.Event()
                here.record()
            landed.append((r0, r1, here))
        # the caller's array is ordinary memory: every chunk is copied out of the recycled pinned buffer as soon as
        # it has landed, by a few threads (NumPy releases the GIL), while the later chunks are still on the bus
        out = np.empty((n, d), dtype=hb.numpy().dtype)
        hb_np = hb.numpy()
        pool = _copy_pool()
        jobs = []
        for r0, r1, here in landed:
            here.synchronize()
            step = max(1, -(-(r1 - r0) // _COPY_THREADS))
            for c0 in range(r0, r1, step):
                c1 = min(r1, c0 + step)
                jobs.append(pool.submit(np.copyto, out[c0:c1], hb_np[c0:c1]))
        for j in jobs:
            j.result()
        main.wait_stream(up)
        return hs.numpy().astype(_score_dtype(d * self.sections)), out

    def packed(self, activations):
        """(scores int32 [N], profile bit-packed [N, sections * W] int32) as CUDA tensors — nothing leaves HBM; feed
        to `prioritizers.cam_from_bits`.  W = `tip_cover_packed_words(D)`; plane s holds section s in NAC's layout
        (libb200tip `tip_kmnc_packed`), and the scores are those of `buckets()`.  Takes what `buckets()` takes.

        The bits take N * sections * W * 4 bytes of HBM (W = 4 * ceil(D / 128)): 91 MB for N = 10 k, D = 36 k and two
        sections, where `buckets()`' int16 ids take 728 MB.  A row of sections * W >= 2^31 words is beyond
        `cam_from_bits` (ValueError before any launch); that many sections stay with `buckets()` / `cam_from_buckets`."""
        import torch

        from .. import _lib
        from .. import engine as E

        act, _, act_np_dtype, stat_dt = self._prepare(activations)
        lib = _lib.load()
        n, d = act.shape
        words = self.sections * int(lib.tip_cover_packed_words(d))
        if words >= 2 ** 31:
            raise ValueError(f"KMNC.packed: {self.sections} sections x {words // self.sections} words per row exceed "
                             "cam_from_bits' 2^31 words; use buckets() and cam_from_buckets")
        dev = E.require_cuda()
        bits = torch.empty((n, words), dtype=torch.int32, device=dev)
        score = torch.empty(n, dtype=torch.int32, device=dev)
        if n == 0:
            return score, bits
        a_dev = E.to_device(act, dev)
        lo_dev, jump_dev = self._device_stats(dev)
        _lib.check(lib.tip_kmnc_packed(E._p(a_dev), E.tip_dtype(act_np_dtype), n, d, E._p(lo_dev), E._p(jump_dev),
                                       E.tip_dtype(stat_dt), self.sections, E._p(bits), E._p(score), E._stream()),
                   "tip_kmnc_packed")
        return score, bits

    PIPELINE_BYTES = 32 << 20
    PIPELINE_CHUNKS = 8

    def _host_buffers(self, n, d, bdt):
        """pinned result buffers, recycled per shape (the bucket ids are the bulk of the D2H traffic of a call)"""
        import torch

        key = (n, d, bdt)
        if getattr(self, "_host_key", None) != key:
            self._host_bucket = torch.empty((n, d), dtype=bdt, pin_memory=True)
            self._host_score = torch.empty(n, dtype=torch.int32, pin_memory=True)
            self._host_key = key
        return self._host_bucket, self._host_score

    def _side_streams(self, dev):
        import torch

        if getattr(self, "_streams", None) is None:
            self._streams = (torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev))
        return self._streams

    def __call__(self, activations: List[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        score, bucket = self.buckets(activations)
        n, d = bucket.shape
        profiles = np.zeros((n, d, self.sections), dtype=bool)
        np.put_along_axis(profiles, np.maximum(bucket, 0).astype(np.int64)[..., None], (bucket >= 0)[..., None], axis=2)
        return score, profiles


_COPY_THREADS = 4
_POOL = None


def _copy_pool():
    global _POOL
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor

        _POOL = ThreadPoolExecutor(max_workers=_COPY_THREADS, thread_name_prefix="tip-copy")
    return _POOL


class NBC(_ThresholdCoverage):
    """Neuron boundary coverage: at or below min - s*std, at or above max + s*std (neuron_coverage.py:97-132);
    profile [N, D, 2]."""

    _mode = 2
    _planes = 2

    def __init__(self, mins, maxs, stds, scaler: float):
        super().__init__()
        lo = np.concatenate([np.asarray(l).flatten() for l in mins])
        hi = np.concatenate([np.asarray(l).flatten() for l in maxs])
        sd = np.concatenate([np.asarray(l).flatten() for l in stds])
        self.min_boundaries, self.max_boundaries = lo - scaler * sd, hi + scaler * sd     # :113-114, same NumPy expressions

    def _bounds(self):
        dt = np.result_type(self.min_boundaries.dtype, self.max_boundaries.dtype)
        return self.min_boundaries.astype(dt), self.max_boundaries.astype(dt), None


class SNAC(_ThresholdCoverage):
    """Strong neuron activation coverage: at or above max + s*std (neuron_coverage.py:135-148)."""

    _mode = 1

    def __init__(self, maxs, stds, scaler: float):
        super().__init__()
        hi = np.concatenate([np.asarray(l).flatten() for l in maxs])
        sd = np.concatenate([np.asarray(l).flatten() for l in stds])
        self.max_boundaries = hi + scaler * sd

    def _bounds(self):
        return None, self.max_boundaries, None


class TKNC(CoverageMethod):
    """Top-k neuron coverage, per layer (neuron_coverage.py:151-173).  Equal activations at the k-th rank:
    the higher index is marked (NumPy's unstable argsort leaves that case open; the reference's own test
    accepts either outcome).  Each layer of d neurons marks `len(range(d)[-k:])` of them, as the reference's slice
    does: every neuron for k = 0 or k >= d, all but the |k| lowest for k < 0."""

    def __init__(self, top_neurons: int):
        super().__init__()
        self.top_neurons = top_neurons

    def _run(self, activations, want_profile: bool, want_bits: bool):
        import torch

        from .. import _lib
        from .. import engine as E

        lib = _lib.load()
        dev = E.require_cuda()
        layers = []
        for layer in activations:
            if isinstance(layer, torch.Tensor):
                flat = layer.reshape(layer.shape[0], -1)
                flat = flat if flat.dtype in (torch.float32, torch.float64) else flat.to(torch.float32)
                layers.append(flat.to(dev).contiguous())
            else:
                flat = np.reshape(layer, (layer.shape[0], -1))
                if flat.dtype not in (np.float32, np.float64):
                    flat = flat.astype(np.result_type(flat.dtype, np.float32))
                layers.append(E.to_device(flat, dev))
        n = layers[0].shape[0]
        total = sum(int(l.shape[1]) for l in layers)
        profile = torch.empty((n, total), dtype=torch.bool, device=dev) if want_profile else None
        words = int(lib.tip_cover_packed_words(total))
        bits = torch.zeros((n, words), dtype=torch.int32, device=dev) if want_bits else None
        off = score = 0
        for l in layers:
            # the reference marks `np.argsort(layer)[..., -k:]`: k = 0 marks every neuron, k < 0 all but the |k| lowest
            count = len(range(int(l.shape[1]))[-int(self.top_neurons):])
            _lib.check(lib.tip_tknc(E._p(l), E.tip_dtype(l.dtype), n, l.shape[1], count, E._p(profile),
                                    total, off, E._p(bits), words, E._stream()), "tip_tknc")
            off += int(l.shape[1])
            score += count
        return score, profile, bits, n, total

    def __call__(self, activations):
        score, profile, _, n, total = self._run(activations, True, False)
        return np.full(n, score, dtype=_score_dtype(total)), profile.cpu().numpy()

    def packed(self, activations):
        import torch

        score, _, bits, n, _ = self._run(activations, False, True)
        return torch.full((n,), score, dtype=torch.int32, device=bits.device), bits
