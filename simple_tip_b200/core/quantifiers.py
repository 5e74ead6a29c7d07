"""The uncertainty quantifiers the study runs beside DeepGini (handler_model.py:23-85,102-173), on the GPU.

uncertainty-wizard 0.2.0's `MaxSoftmax`, `PredictionConfidenceScore`, `SoftmaxEntropy` and `VariationRatio`, with
its class-method surface (`aliases`, `takes_samples`, `is_confidence`, `problem_type`, `calculate`,
`cast_conf_or_unc`).  `calculate` takes softmax outputs — a NumPy array or a CUDA tensor (float16 / bfloat16 CUDA
tensors are widened to float32) — and returns NumPy arrays: the prediction as int64 and the quantity in the input
dtype (float64 for VariationRatio).  The quantity is unsigned, as uwiz's `calculate` returns it; the study stores
`cast_conf_or_unc(as_confidence=False, ...)` of it, i.e. the negated max softmax and PCS.

    MaxSoftmax                 max_c p                                   confidence   bit-identical to NumPy
    PredictionConfidenceScore  top-1 minus top-2 of p                    confidence   bit-identical
    SoftmaxEntropy             -sum q*log2(q), q = p with 0 -> 1e-20     uncertainty  NumPy's summation order
    VariationRatio             1 - (votes of the mode) / S over S        uncertainty  bit-identical
                               samples [N, S, C]

The prediction is np.argmax of each row (the first maximum; the first NaN if the row holds one, and then every
quantity of the row is NaN); a sample's vote is np.argmax of the sample, and VariationRatio's prediction is the lowest
class with the most votes (scipy.stats.mode).  The semantics are restated from uncertainty-wizard 0.2.0, which is not
a dependency.
"""
from __future__ import annotations

from typing import List

import numpy as np

from .deepgini import _CLASSIFICATION, _Base, device_probs


def _softmax_stat(nn_outputs, kind: int):
    import torch

    from .. import _lib
    from .. import engine as E

    p_dev, p_np_dtype = device_probs(nn_outputs, 2)
    n, c = p_dev.shape
    if kind == _lib.STAT_PCS and c < 2:
        raise ValueError("PredictionConfidenceScore needs at least two classes")
    lib = _lib.load()
    pred = torch.empty(n, dtype=torch.int32, device=p_dev.device)
    out = torch.empty(n, dtype=p_dev.dtype, device=p_dev.device)
    _lib.check(lib.tip_softmax_stat(E._p(p_dev), E.tip_dtype(p_np_dtype), n, c, kind, E._p(pred), E._p(out),
                                    E._stream()), "tip_softmax_stat")
    return pred.cpu().numpy().astype(np.int64), out.cpu().numpy()


class MaxSoftmax(_Base):
    """Max softmax - confidence (the largest softmax output)."""

    @classmethod
    def aliases(cls) -> List[str]:
        return ["softmax", "MaxSoftmax", "max_softmax", "SM"]

    @classmethod
    def takes_samples(cls) -> bool:
        return False

    @classmethod
    def is_confidence(cls) -> bool:
        return True

    @classmethod
    def problem_type(cls):
        return _CLASSIFICATION

    @classmethod
    def calculate(cls, nn_outputs):
        from .. import _lib

        return _softmax_stat(nn_outputs, _lib.STAT_MAX)


class PredictionConfidenceScore(_Base):
    """Prediction confidence score - confidence (largest minus second largest softmax output)."""

    @classmethod
    def aliases(cls) -> List[str]:
        return ["pcs", "PredictionConfidenceScore", "prediction_confidence_score", "PCS"]

    @classmethod
    def takes_samples(cls) -> bool:
        return False

    @classmethod
    def is_confidence(cls) -> bool:
        return True

    @classmethod
    def problem_type(cls):
        return _CLASSIFICATION

    @classmethod
    def calculate(cls, nn_outputs):
        from .. import _lib

        return _softmax_stat(nn_outputs, _lib.STAT_PCS)


class SoftmaxEntropy(_Base):
    """Softmax entropy - uncertainty (base-2 entropy of the softmax outputs)."""

    @classmethod
    def aliases(cls) -> List[str]:
        return ["softmax_entropy", "SoftmaxEntropy", "SE"]

    @classmethod
    def takes_samples(cls) -> bool:
        return False

    @classmethod
    def is_confidence(cls) -> bool:
        return False

    @classmethod
    def problem_type(cls):
        return _CLASSIFICATION

    @classmethod
    def calculate(cls, nn_outputs):
        from .. import _lib

        return _softmax_stat(nn_outputs, _lib.STAT_ENTROPY)


class VariationRatio(_Base):
    """Variation ratio - uncertainty (share of the samples that do not vote for the mode), over [N, S, C]
    sampled softmax outputs."""

    @classmethod
    def aliases(cls) -> List[str]:
        return ["variation_ratio", "VariationRatio", "var_ratio", "VR"]

    @classmethod
    def takes_samples(cls) -> bool:
        return True

    @classmethod
    def is_confidence(cls) -> bool:
        return False

    @classmethod
    def problem_type(cls):
        return _CLASSIFICATION

    @classmethod
    def calculate(cls, nn_outputs):
        p_dev, _ = device_probs(nn_outputs, 3)
        n, s, c = p_dev.shape
        votes = Votes(n, c, p_dev.device)
        votes.add(p_dev, s, sample_stride=c, row_stride=s * c)
        return votes.finish(s)


class Votes:
    """Running argmax vote counts of n rows over c classes (int32 [n, c] in HBM), fed sample chunk by sample chunk
    (`tip_vote_add`), then reduced to (mode, variation ratio) (`tip_vote_finish`).  `device` must be the current CUDA
    device, on whose stream the kernels run."""

    def __init__(self, n: int, c: int, device):
        import torch

        from .. import engine as E

        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = E.require_cuda()
        if device != E.require_cuda():
            raise ValueError(f"vote counts must live on the current CUDA device {E.require_cuda()}, not {device}")
        self.n, self.c = n, c
        self.counts = torch.zeros((n, c), dtype=torch.int32, device=device)

    def add(self, probs, samples: int, sample_stride: int, row_stride: int, row0: int = 0, rows: int = None):
        """Votes of `samples` samples of rows [row0, row0 + rows); sample s of row i (relative to row0) is the
        c-vector at element i * row_stride + s * sample_stride from the first element of `probs`, a float32 / float64
        CUDA tensor on the counts' device (a view is fine: only its storage bounds the elements addressed).
        Raises ValueError for anything else, before any launch."""
        import torch

        from .. import _lib
        from .. import engine as E

        rows = self.n - row0 if rows is None else rows
        if not (0 <= row0 and 0 <= rows and row0 + rows <= self.n and samples >= 0 and sample_stride >= 0
                and row_stride >= 0):
            raise ValueError(f"rows [{row0}, {row0 + rows}) of {self.n}, {samples} samples, strides "
                             f"({sample_stride}, {row_stride}): out of range")
        if not isinstance(probs, torch.Tensor) or probs.device != self.counts.device:
            where = probs.device if isinstance(probs, torch.Tensor) else type(probs).__name__
            raise ValueError(f"probs must be a CUDA tensor on {self.counts.device}, got {where}")
        if probs.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"probs must be float32 or float64, got {probs.dtype}")
        if rows == 0 or samples == 0:
            return
        last = (rows - 1) * row_stride + (samples - 1) * sample_stride + self.c      # one past the last element read
        avail = probs.untyped_storage().nbytes() // probs.element_size() - probs.storage_offset()
        if last > avail:
            raise ValueError(f"the votes would read {last} elements of probs, its storage holds {avail}")
        counts = self.counts[row0:row0 + rows]
        _lib.check(_lib.load().tip_vote_add(E._p(probs), E.tip_dtype(probs.dtype), rows, self.c, samples,
                                            sample_stride, row_stride, E._p(counts), E._stream()), "tip_vote_add")

    def finish(self, samples: int):
        """(pred int64, vr float64) as NumPy arrays, `samples` being the number of votes every row received."""
        import torch

        from .. import _lib
        from .. import engine as E

        if self.n and samples < 1:
            raise ValueError("VariationRatio needs at least one sample")
        pred = torch.empty(self.n, dtype=torch.int32, device=self.counts.device)
        vr = torch.empty(self.n, dtype=torch.float64, device=self.counts.device)
        _lib.check(_lib.load().tip_vote_finish(E._p(self.counts), self.n, self.c, max(samples, 1), E._p(pred),
                                               E._p(vr), E._stream()), "tip_vote_finish")
        return pred.cpu().numpy().astype(np.int64), vr.cpu().numpy()
