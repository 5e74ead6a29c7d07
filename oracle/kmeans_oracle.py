"""float64 reference of the device k-means (simple_tip_b200/csrc/kmeans.cu) (TEST INFRASTRUCTURE ONLY).

Written from sklearn's algorithm (`sklearn.cluster._kmeans._kmeans_plusplus` and `_kmeans_single_lloyd`,
`_k_means_common._relocate_empty_clusters_dense`), not from the CUDA: greedy k-means++ seeding, Lloyd iterations,
empty-cluster relocation and the three stopping rules.  Where sklearn draws from its RandomState this module uses
the device's counter RNG instead (`km_uniform`), so every run of a device fit has one fully determined trajectory
that this module reproduces.  The relocation rule is the one DESIGN.md §9 states:

  * the set of empty clusters is fixed before any row moves; they are filled in ascending cluster order with the
    rows farthest from their centres, in descending order of that distance (ties: lowest row index);
  * relocation is skipped when every row sits exactly on its centre (more clusters than distinct rows);
  * a cluster that is still empty keeps its previous centre.

Every decision of a run (a draw, the kept trial, a row's nearest centre, the relocated rows, the tol test) comes
with a margin: how far, relative to the quantities compared, the decision is from going the other way.  A test
compares a device run exactly only when all of its margins exceed the device's rounding error.

Inputs are NumPy arrays; nothing in the product package imports this module.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List

import numpy as np

MASK64 = (1 << 64) - 1


# ---- the device's counter RNG: splitmix64 over (seed, k, run, step, trial) -----------------------------------------
def km_mix(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def km_uniform(seed: int, k: int, run: int, step: int, trial: int) -> float:
    h = km_mix(seed & MASK64)
    for v in (k, run, step, trial):
        h = km_mix(h ^ (v & MASK64))
    return (h >> 11) * 2.0 ** -53


def n_local_trials(k: int) -> int:
    return 2 + int(math.log(k))


def exact_grid(*arrays) -> bool:
    """True when every value is a multiple of 1/8 small enough that every squared distance between them, in fp32,
    and every sum of n such distances, in double, is exact: then any summation order gives the same bits, and
    every tie is exact on the device too."""
    n = max(a.shape[0] for a in arrays)
    d = arrays[0].shape[1]
    m = 0.0
    for a in arrays:
        s = np.asarray(a, dtype=np.float64) * 8.0
        if not np.array_equal(s, np.round(s)):
            return False
        m = max(m, float(np.abs(s).max()))
    return d * (2 * m) ** 2 < 2.0 ** 24 and n * d * (2 * m) ** 2 < 2.0 ** 50


def _rel_gap(a: float, b: float) -> float:
    """|a - b| relative to the larger of the two (0 when both are 0)"""
    s = max(abs(a), abs(b))
    return abs(a - b) / s if s > 0 else 0.0


# ---- k-means++ -----------------------------------------------------------------------------------------------------
@dataclass
class Seeding:
    idx: np.ndarray                                         # [k] seed row indices
    draw_margins: List[float] = field(default_factory=list)  # per draw: gap of the target to the cumulative sums
    trial_margins: List[float] = field(default_factory=list)  # per step: gap between the best and next potential

    @property
    def margin(self) -> float:
        return min(self.draw_margins + self.trial_margins, default=math.inf)


def _draw(closest: np.ndarray, cum: np.ndarray, target: float, pot: float):
    """First row whose cumulative D^2 reaches target, rows with D^2 = 0 never (np.searchsorted on the cumulative
    sum); if no row qualifies, the last row with D^2 > 0, or row 0 if there is none.  Returns (row, margin)."""
    pos = closest > 0
    ok = pos & (cum >= target)
    if ok.any():
        i = int(np.argmax(ok))
        below = cum[i] - closest[i]
        return i, min(target - below, cum[i] - target) / pot
    if pos.any():   # the target lies past the total: only rounding gets here, so the decision has no margin
        return int(np.flatnonzero(pos)[-1]), 0.0
    return 0, math.inf


def kmeanspp(x: np.ndarray, k: int, seed: int, run: int) -> Seeding:
    """sklearn's greedy `_kmeans_plusplus` in float64 with n_local_trials = 2 + int(log(k)), on the device's
    draws: the first centre is row min(n-1, floor(u(0, 0) * n)); trial t of step s targets u(s, t) * potential;
    the kept trial has the lowest potential (ties: lowest trial)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    trials = n_local_trials(k)
    exact = exact_grid(x)   # every potential and cumulative sum exact: no decision depends on rounding
    cache = {}

    def d2(i):
        if i not in cache:
            cache[i] = ((x - x[i]) ** 2).sum(axis=1)
        return cache[i]

    first = min(n - 1, int(km_uniform(seed, k, run, 0, 0) * n))
    out = Seeding(idx=np.empty(k, dtype=np.int64))
    out.idx[0] = first
    closest = d2(first)
    pot = float(closest.sum())
    for step in range(1, k):
        cum = np.cumsum(closest)
        cands, pots, dists = [], [], []
        for t in range(trials):
            c, m = _draw(closest, cum, km_uniform(seed, k, run, step, t) * pot, pot)
            out.draw_margins.append(math.inf if exact else m)
            dt = np.minimum(closest, d2(c))
            cands.append(c)
            dists.append(dt)
            pots.append(float(dt.sum()))
        best = int(np.argmin(pots))   # first minimum
        # a trial whose candidate has the best candidate's values ties exactly on every device as well
        others = [pots[t] for t in range(trials) if not np.array_equal(x[cands[t]], x[cands[best]])]
        if not exact:
            out.trial_margins.append(min((_rel_gap(p, pots[best]) for p in others), default=math.inf))
        out.idx[step] = cands[best]
        closest, pot = dists[best], pots[best]
    return out


# ---- Lloyd -----------------------------------------------------------------------------------------------------------
@dataclass
class LloydRun:
    centres: np.ndarray          # [k, d] float64 values of the final centres (rounded to the input dtype)
    labels: np.ndarray           # [n] final labels: one more assignment pass with the final centres
    inertia: float
    n_iter: int
    stop: str                    # "strict", "tol", "max_iter" or "none" (max_iter = 0)
    iter_labels: List[np.ndarray] = field(default_factory=list)   # labels of every iteration's assignment
    assign_margins: List[np.ndarray] = field(default_factory=list)  # per assignment pass (final pass last): per row
    relocations: List[dict] = field(default_factory=list)          # per relocation: iteration, moves, margin
    tol_margins: List[float] = field(default_factory=list)

    @property
    def margin(self) -> float:
        m = [float(a.min()) for a in self.assign_margins if a.size]
        m += [r["margin"] for r in self.relocations] + self.tol_margins
        return min(m, default=math.inf)


class _Assigner:
    """Nearest centre of every row, ties to the lowest index.  Distances for the argmin come from the expansion
    |x|^2 + |c|^2 - 2<x, c> on rows centred on their mean (good to ~1e-13 of the data's spread, far below every
    margin a test accepts); the distance of each row to its own centre is recomputed from the differences."""

    def __init__(self, x: np.ndarray):
        self.x = x
        self.mu = x.mean(axis=0)
        self.xc = x - self.mu
        self.xn = (self.xc ** 2).sum(axis=1)

    def __call__(self, cen: np.ndarray):
        cc = cen - self.mu
        d = self.xn[:, None] + (cc ** 2).sum(axis=1)[None, :] - 2.0 * (self.xc @ cc.T)
        k = cen.shape[0]
        # a centre equal to an earlier one never wins (ties go to the lowest index) and is no competitor either
        for c in range(1, k):
            if any(np.array_equal(cen[c], cen[e]) for e in range(c)):
                d[:, c] = np.inf
        lab = np.argmin(d, axis=1)
        if k > 1:
            part = np.partition(d, 1, axis=1)
            d1, d2 = part[:, 0], part[:, 1]
            with np.errstate(invalid="ignore", divide="ignore"):
                margin = np.where(np.isinf(d2), np.inf, (d2 - d1) / np.maximum(d2, 1e-300))
        else:
            margin = np.full(lab.shape, np.inf)
        return lab.astype(np.int32), margin

    def own_dist(self, cen: np.ndarray, lab: np.ndarray) -> np.ndarray:
        return ((self.x - cen[lab]) ** 2).sum(axis=1)


def _relocate(x, dist, lab, sums, cnt):
    """Empty clusters (fixed before any row moves) take the farthest rows, descending, ties to the lowest row;
    skipped when every distance is 0.  Updates sums / cnt in place; returns the record of what moved."""
    empty = np.flatnonzero(cnt == 0)
    if empty.size == 0 or dist.max() == 0.0:
        return None if empty.size == 0 else {"moves": [], "margin": math.inf, "empty": empty.tolist()}
    order = np.lexsort((np.arange(dist.shape[0]), -dist))
    far = order[: empty.size]
    margin = math.inf
    for j in range(min(empty.size + 1, order.size) - 1):   # the picks' order and the last pick against the next row
        a, b = order[j], order[j + 1]
        if dist[a] == dist[b] and lab[a] == lab[b] and np.array_equal(x[a], x[b]):
            continue   # identical rows on the same centre: an exact tie everywhere, broken by the row index
        margin = min(margin, _rel_gap(dist[a], dist[b]))
    moves = []
    for c, r in zip(empty, far):
        donor = int(lab[r])
        sums[donor] -= x[r]
        sums[c] = x[r]
        cnt[donor] -= 1
        cnt[c] = 1
        moves.append((int(c), int(r), donor))
    return {"moves": moves, "margin": margin, "empty": empty.tolist()}


def _tol_margin(x, lab, sums, old, new, shift, tol_abs, dtype, moved) -> float:
    """Margin of the test shift <= tol_abs.  Centres computed in another summation order may differ from these in
    the last bit of the stored dtype, so a shift within that rounding of tol_abs has no margin, with one
    exception: a shift of exactly 0 from member sums that are exact (every order gives them) is 0 everywhere."""
    if shift == 0.0 and not moved:
        exact = all(math.fsum(x[lab == c, j]) == sums[c, j] for c in np.unique(lab) for j in range(x.shape[1]))
        if exact:
            return math.inf
    ulp = 2.0 * np.finfo(dtype).eps * max(float(np.abs(new).max()), float(np.abs(old).max()))
    floor = new.size * ulp * ulp
    s = max(shift, tol_abs, floor)
    return abs(shift - tol_abs) / s if s > 0 else 0.0


def lloyd(x: np.ndarray, seeds: np.ndarray, max_iter: int, tol_abs: float, dtype=np.float64) -> LloydRun:
    """sklearn's `_kmeans_single_lloyd` in float64 from the centres `seeds` ([k, d] values): labels start at -1;
    each iteration assigns every row to its nearest centre, relocates empty clusters and moves every centre to
    the mean of its members (rounded to `dtype`, the dtype the device stores centres in); a run stops when no
    label changed, else when sum ||shift||^2 <= tol_abs, else after max_iter iterations (n_iter = i + 1).  The
    final labels and inertia come from one more assignment pass."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    cen = np.asarray(seeds, dtype=np.float64).copy()
    k = cen.shape[0]
    asg = _Assigner(x)
    prev = np.full(n, -1, dtype=np.int32)
    run = LloydRun(centres=cen, labels=prev, inertia=0.0, n_iter=0, stop="none")
    for it in range(max_iter):
        lab, margin = asg(cen)
        run.iter_labels.append(lab)
        run.assign_margins.append(margin)
        cnt = np.bincount(lab, minlength=k).astype(np.int64)
        sums = np.zeros_like(cen)
        np.add.at(sums, lab, x)
        moved = False
        if (cnt == 0).any():
            rec = _relocate(x, asg.own_dist(cen, lab), lab, sums, cnt)
            rec["iteration"] = it
            run.relocations.append(rec)
            moved = bool(rec["moves"])
        new = cen.copy()
        full = cnt > 0
        new[full] = (sums[full] / cnt[full, None]).astype(dtype).astype(np.float64)
        shift = float(((new - cen) ** 2).sum())
        run.n_iter = it + 1
        if np.array_equal(lab, prev):
            cen = new
            run.stop = "strict"
            break
        run.tol_margins.append(_tol_margin(x, lab, sums, cen, new, shift, tol_abs, dtype, moved))
        cen = new
        if shift <= tol_abs:
            run.stop = "tol"
            break
        prev = lab
    else:
        if max_iter > 0:
            run.stop = "max_iter"
    run.centres = cen
    run.labels, margin = asg(cen)
    run.assign_margins.append(margin)
    run.inertia = float(asg.own_dist(cen, run.labels).sum())
    return run


# ---- a whole fit -----------------------------------------------------------------------------------------------------
@dataclass
class Fit:
    seedings: List[Seeding]
    runs: List[LloydRun]
    best: int

    @property
    def inertia(self) -> np.ndarray:
        return np.array([r.inertia for r in self.runs])


def fit(x: np.ndarray, k: int, runs: int, seed: int, max_iter: int, tol_abs: float, dtype=None) -> Fit:
    """Every run of a device fit (tip_kmeans_fit with the same seed, max_iter and absolute tol) and the best run
    by inertia (first minimum).  dtype: the input's dtype (default: x's), in which centres are stored."""
    dtype = np.dtype(dtype if dtype is not None else np.asarray(x).dtype)
    x64 = np.asarray(x, dtype=np.float64)
    seedings = [kmeanspp(x64, k, seed, r) for r in range(runs)]
    out = [lloyd(x64, x64[s.idx], max_iter, tol_abs, dtype) for s in seedings]
    inertia = np.array([r.inertia for r in out])
    return Fit(seedings, out, int(np.argmin(inertia)))
