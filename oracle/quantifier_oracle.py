"""NumPy restatement of the uncertainty quantifiers the study runs beside DeepGini (TEST INFRASTRUCTURE ONLY).

Provenance caveat: uncertainty-wizard 0.2.0 is not installed here and cannot be installed offline, so — like the
`uncertainty_wizard` stub of `ref_harness.py` (SURVEY.md §8(c)) — the semantics below are restated from memory of
that package, not read from its source.  Two details in particular are as recalled and should be re-checked against
uwiz whenever it is available:

  * SoftmaxEntropy uses base 2 (np.log2), and
  * it replaces exact zeros of the softmax output by 1e-20 (in the input dtype) before taking the logarithm.
    Where a row holds such zeros the substitution moves the entropy by at most about C * 6.6e-19.

Contract (input `p [N, C]`, float32 or float64, C-contiguous; `pred = np.argmax(p, axis=1)`, first index on ties):

  max_softmax(p)      np.max(p, axis=1)                                        confidence
  pcs(p)              s = np.sort(p, axis=1); s[:, -1] - s[:, -2]              confidence; C = 1 -> ValueError
  softmax_entropy(p)  -np.sum(q * np.log2(q), axis=1), q = p, 0 -> 1e-20       uncertainty; p is not modified
  variation_ratio(p)  p [N, S, C]; votes = argmax over C per sample; pred = the lowest class with the most votes
                      (scipy.stats.mode's tie rule); vr = 1 - max_votes / S in float64          uncertainty

NaN follows NumPy, whose functions these are:
  * pred and every vote are np.argmax's: a NaN beats any number, and the first NaN wins;
  * max_softmax is NaN on a row with a NaN (np.max propagates it);
  * pcs is NaN on such a row (np.sort puts NaN last, so s[:, -1] is NaN), and so is the entropy (the sum propagates);
  * a row with two +inf has pcs inf - inf = NaN; a row of -inf has pcs NaN and max -inf.

`cast_conf_or_unc(as_confidence, scores)` negates a confidence when an uncertainty is asked for (the study calls
with as_confidence=False, so it stores -max_softmax and -pcs).
"""
from __future__ import annotations

import numpy as np


def _check(p, ndim):
    p = np.asarray(p)
    assert p.ndim == ndim and p.dtype in (np.float32, np.float64)
    return p


def max_softmax(p):
    p = _check(p, 2)
    return np.argmax(p, axis=1), np.max(p, axis=1)


def pcs(p):
    p = _check(p, 2)
    if p.shape[1] < 2:
        raise ValueError("PredictionConfidenceScore needs at least two classes")
    s = np.sort(p, axis=1)
    return np.argmax(p, axis=1), s[:, -1] - s[:, -2]


def softmax_entropy(p):
    p = _check(p, 2)
    q = p.copy()
    q[q == 0] = p.dtype.type(1e-20)
    return np.argmax(p, axis=1), -np.sum(q * np.log2(q), axis=1)


def vote_counts(p):
    """[N, S, C] samples -> int64 [N, C] argmax votes."""
    p = _check(p, 3)
    n, s, c = p.shape
    votes = np.argmax(p, axis=2)
    counts = np.zeros((n, c), dtype=np.int64)
    np.add.at(counts, (np.repeat(np.arange(n), s), votes.reshape(-1)), 1)
    return counts


def variation_ratio(p):
    p = _check(p, 3)
    counts = vote_counts(p)
    pred = np.argmax(counts, axis=1)                       # lowest class among the most voted
    max_votes = counts[np.arange(p.shape[0]), pred] if p.shape[0] else np.zeros(0, dtype=np.int64)
    return pred, 1 - max_votes / p.shape[1]


def cast_conf_or_unc(is_confidence: bool, as_confidence, scores):
    if as_confidence is not None and is_confidence != as_confidence:
        return scores * -1
    return scores


def study_uncertainties(p, samples=None):
    """The values the study stores (handler_model.py:141-166, as_confidence=False): {softmax, pcs,
    softmax_entropy, deep_gini[, VR]}."""
    from . import np_oracle

    out = {"softmax": cast_conf_or_unc(True, False, max_softmax(p)[1]),
           "pcs": cast_conf_or_unc(True, False, pcs(p)[1]),
           "softmax_entropy": softmax_entropy(p)[1],
           "deep_gini": np_oracle.deepgini_oracle(p)[1]}
    if samples is not None:
        out["VR"] = variation_ratio(samples)[1]
    return out
