"""The surprise-coverage CAM order in closed form, restated in NumPy (handler_surprise.py:101-115 over
prioritizers.py:16-59).

`SurpriseCoverageMapper(sections, ub).get_coverage_profile(v)` sets profile[i, b] = t[b] <= v[i] < t[b+1].  For
NaN-free, non-decreasing thresholds the buckets are disjoint, so a row holds at most one True.  Then a sample's
gain in `cam` is 1 while its bucket is uncovered and 0 after; `np.argmax` takes the lowest index with gain 1, and
covering its bucket zeroes every other sample of that bucket.  By induction the greedy picks are the first sample
of every non-empty bucket, in ascending sample order; the tail is `np.argsort(-scores)` over the rest, as in
`np_oracle.cam_oracle`.  Tests check this against `np_oracle.cam_oracle` on the dense profile.
"""
from __future__ import annotations

import numpy as np


def sc_buckets(values: np.ndarray, thresholds: np.ndarray) -> np.ndarray:
    """Bucket of every value (-1: none), for non-decreasing thresholds; values compared in float64 as NumPy
    promotes float32 against the mapper's float64 thresholds.  NaN lies in no bucket."""
    t = np.asarray(thresholds, dtype=np.float64)
    v = np.asarray(values).astype(np.float64)
    b = np.searchsorted(t, v, side="right") - 1          # number of thresholds <= v, minus one (NaN sorts last)
    b[(b < 0) | (b >= t.shape[0] - 1)] = -1
    ok = b >= 0
    inside = np.zeros_like(ok)
    inside[ok] = (t[b[ok]] <= v[ok]) & (v[ok] < t[b[ok] + 1])
    b[~inside] = -1
    return b


def sc_cam_oracle(scores: np.ndarray, thresholds: np.ndarray) -> np.ndarray:
    """cam(scores, SurpriseCoverageMapper's profile of scores) for NaN-free, non-decreasing thresholds."""
    scores = np.asarray(scores).copy()
    b = sc_buckets(scores, thresholds)
    covered = np.flatnonzero(b >= 0)
    _, first = np.unique(b[covered], return_index=True)
    greedy = np.sort(covered[first])
    order = [int(i) for i in greedy]
    if scores.shape[0]:
        floor = np.min(scores) - 1                        # prioritizers.py:48-52
        scores[greedy] = floor - 1
        for x in np.argsort(-scores):
            if scores[x] < floor:
                break
            order.append(int(x))
    return np.array(order, dtype=np.int64)
