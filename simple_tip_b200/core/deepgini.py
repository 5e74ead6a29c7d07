"""DeepGini behind the reference's `src.core.deepgini` API (deepgini.py:12-40).

`calculate` returns (argmax class, 1 - sum_c p^2) from libb200tip.so; the sum of squares uses
NumPy's pairwise order so float32 and float64 results are bit-identical to
`1 - np.sum(p * p, axis=1)`.  When `uncertainty_wizard` is installed DeepGini subclasses its
`Quantifier` (so `handler_model.py:17` can register it); otherwise a structural stand-in with
the same class-method surface is used.
"""
from __future__ import annotations

from typing import List

import numpy as np

try:  # pragma: no cover - depends on the host environment
    import uncertainty_wizard as uwiz

    _Base = uwiz.quantifiers.Quantifier
    _CLASSIFICATION = uwiz.ProblemType.CLASSIFICATION
except Exception:  # uncertainty-wizard is optional
    uwiz = None

    class _Base:  # same surface as uwiz.quantifiers.Quantifier's class methods
        @classmethod
        def cast_conf_or_unc(cls, as_confidence, superv_scores):
            if as_confidence is not None and cls.is_confidence() != as_confidence:
                return superv_scores * -1
            return superv_scores

    _CLASSIFICATION = 2


class DeepGini(_Base):
    """DeepGini - uncertainty (1 minus sum of squared softmax outputs)."""

    @classmethod
    def aliases(cls) -> List[str]:
        return ["custom::deep_gini"]

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
    def calculate(cls, nn_outputs: np.ndarray):
        import torch

        from .. import _lib
        from .. import engine as E

        p_dev, p_np_dtype = device_probs(nn_outputs, 2)
        lib = _lib.load()
        n, c = p_dev.shape
        pred = torch.empty(n, dtype=torch.int32, device=p_dev.device)
        gini = torch.empty(n, dtype=p_dev.dtype, device=p_dev.device)
        _lib.check(lib.tip_deepgini(E._p(p_dev), E.tip_dtype(p_np_dtype), n, c, E._p(pred), E._p(gini), E._stream()),
                   "tip_deepgini")
        return pred.cpu().numpy().astype(np.int64), gini.cpu().numpy()


def device_probs(nn_outputs, ndim: int):
    """Softmax outputs as a contiguous float32 / float64 CUDA tensor, and their NumPy dtype.  CUDA tensors stay in
    HBM (float16 / bfloat16 ones are widened to float32); host arrays keep float32 / float64 and are otherwise
    widened to float64, then uploaded."""
    import torch

    from .. import engine as E

    if isinstance(nn_outputs, torch.Tensor) and nn_outputs.is_cuda:     # softmax outputs already in HBM
        p = nn_outputs if nn_outputs.dtype in (torch.float32, torch.float64) else nn_outputs.to(torch.float32)
        p_np_dtype = E.NP_DTYPE[p.dtype]
    else:
        p = np.asarray(nn_outputs)
        if p.dtype not in (np.float32, np.float64):
            p = p.astype(np.float64)
        p_np_dtype = p.dtype
    assert p.ndim == ndim, "nn_outputs must be (samples, classes)" if ndim == 2 else \
        "nn_outputs must be (samples, sample_size, classes)"
    return E.to_device(p, E.require_cuda()), p_np_dtype
