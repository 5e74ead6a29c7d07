"""CPU tests of the float64 k-means reference (oracle/kmeans_oracle.py) that the device k-means is compared
against: its RNG port, its Lloyd iterations against sklearn's own, and its relocation rule on hand-built cases."""
import math

import numpy as np
import pytest

from oracle import kmeans_oracle as KO


def test_km_mix_is_splitmix64():
    assert KO.km_mix(0) == 0xE220A8397B1DCDAF            # splitmix64's first output for state 0
    assert KO.km_mix(KO.MASK64) == KO.km_mix(0xFFFFFFFFFFFFFFFF)
    assert all(0 <= KO.km_mix(v) <= KO.MASK64 for v in (1, 2 ** 63, 0x9E3779B97F4A7C15))


def test_km_uniform_pinned_values():
    # key order (seed, k, run, step, trial); values cross-checked against a C build of kmeans.cu's km_uniform
    assert KO.km_uniform(0, 1, 0, 0, 0) == 0.9752873302169826
    assert KO.km_uniform(0, 5, 3, 2, 1) == 0.912536289366515
    assert KO.km_uniform(7, 64, 63, 63, 5) == 0.42046013358880274
    assert KO.km_uniform(2 ** 64 - 1, 2, 0, 1, 0) == 0.33967217750753564
    u = [KO.km_uniform(3, 4, r, s, t) for r in range(4) for s in range(4) for t in range(3)]
    assert all(0.0 <= v < 1.0 for v in u) and len(set(u)) == len(u)


def test_n_local_trials_is_sklearns():
    assert [KO.n_local_trials(k) for k in (1, 2, 3, 7, 8, 20, 21, 54, 55, 64)] == [2, 2, 3, 3, 4, 4, 5, 5, 6, 6]


def _blobs(n, d, k, seed, spread):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(k, d)) * spread
    return centres[rng.integers(0, k, size=n)] + rng.normal(size=(n, d))


def _sklearn_lloyd(x, seeds, max_iter, tol):
    from sklearn.cluster import KMeans

    km = KMeans(seeds.shape[0], init=seeds, n_init=1, algorithm="lloyd", max_iter=max_iter, tol=tol).fit(x)
    return km


@pytest.mark.parametrize("case, max_iter, tol", [
    ("blobs", 300, 1e-4), ("blobs", 300, 0.0), ("overlap", 300, 1e-4), ("overlap", 300, 0.0),
    ("overlap", 1, 1e-4), ("overlap", 2, 1e-4), ("overlap", 2, 0.0)])
def test_lloyd_matches_sklearn(case, max_iter, tol):
    if case == "blobs":
        x, k = _blobs(600, 5, 4, seed=1, spread=5.0), 4
    else:
        x, k = np.random.default_rng(2).normal(size=(800, 3)), 6   # one Gaussian cut into 6: many iterations
    seeds = x[KO.kmeanspp(x, k, seed=11, run=0).idx]
    tol_abs = float(np.mean(np.var(x, axis=0))) * tol
    run = KO.lloyd(x, seeds, max_iter, tol_abs)
    sk = _sklearn_lloyd(x, seeds, max_iter, tol)
    assert not run.relocations and run.margin > 1e-9
    assert run.n_iter == sk.n_iter_
    assert np.array_equal(run.labels, sk.labels_)
    np.testing.assert_allclose(run.centres, sk.cluster_centers_, rtol=1e-12, atol=1e-12)
    assert math.isclose(run.inertia, sk.inertia_, rel_tol=1e-12)
    if case == "overlap" and max_iter == 300:
        assert run.n_iter > 10 and (tol > 0 or run.stop == "strict")
    if max_iter <= 2:
        assert run.stop == "max_iter" and len(run.iter_labels) == max_iter


def test_kmeanspp_draws_follow_the_cumulative_potential():
    x = np.array([[0.0], [0.0], [1.0], [3.0], [3.0], [10.0]])
    s = KO.kmeanspp(x, 3, seed=5, run=2)
    # replay the draws by hand: first centre uniform, then every trial on searchsorted of the cumulative D^2
    first = min(5, int(KO.km_uniform(5, 3, 2, 0, 0) * 6))
    assert s.idx[0] == first
    closest = ((x - x[first]) ** 2).sum(1)
    for step in (1, 2):
        pot = closest.sum()
        cum = np.cumsum(closest)
        pots, dists, cands = [], [], []
        for t in range(KO.n_local_trials(3)):
            target = KO.km_uniform(5, 3, 2, step, t) * pot
            c = int(np.searchsorted(cum, target, side="left"))
            while closest[c] == 0:   # a zero-D^2 row shares its cumulative sum with the row before it
                c += 1
            dt = np.minimum(closest, ((x - x[c]) ** 2).sum(1))
            cands.append(c), dists.append(dt), pots.append(dt.sum())
        b = int(np.argmin(pots))
        assert s.idx[step] == cands[b]
        closest = dists[b]
    assert len(set(s.idx.tolist())) == 3


def test_kmeanspp_with_no_potential_left_picks_row_zero():
    x = np.repeat(np.array([[1.0, 2.0], [4.0, -1.0]]), 3, axis=0)   # 2 distinct rows, k = 4
    s = KO.kmeanspp(x, 4, seed=0, run=0)
    assert {tuple(x[i]) for i in s.idx[:2]} == {(1.0, 2.0), (4.0, -1.0)}
    assert s.idx[2] == 0 and s.idx[3] == 0
    assert s.margin > 0
    xs = np.full((9, 3), 0.25)                                       # every row equal
    s = KO.kmeanspp(xs, 3, seed=4, run=1)
    assert s.idx[0] == min(8, int(KO.km_uniform(4, 3, 1, 0, 0) * 9)) and s.idx[1] == 0 and s.idx[2] == 0


def test_relocation_leaves_an_emptied_singleton_donor_empty():
    # rows 0, 0.1, 0.3 go to centre 1; row 12 alone to centre 2; centre 0 is empty.  The farthest row (12, 64 from
    # its centre) is the only member of cluster 2, which has a higher index: it moves to cluster 0, and cluster 2,
    # emptied by the move, is not refilled in the same iteration and keeps its centre.
    x = np.array([[0.0], [0.1], [0.3], [12.0]])
    seeds = np.array([[-50.0], [0.0], [20.0]])
    run = KO.lloyd(x, seeds, max_iter=1, tol_abs=0.0)
    assert run.iter_labels[0].tolist() == [1, 1, 1, 2]
    assert run.relocations[0]["moves"] == [(0, 3, 2)]
    np.testing.assert_array_equal(run.centres[:, 0], [12.0, np.float64(0.4) / 3, 20.0])
    # iteration 2: 12 -> cluster 0, cluster 2 empty again: its farthest row (0.3, from 0.4/3) is taken; the rows at 0
    # and 0.1 do not tie with it
    run = KO.lloyd(x, seeds, max_iter=2, tol_abs=0.0)
    assert run.iter_labels[1].tolist() == [1, 1, 1, 0]
    assert run.relocations[1]["moves"] == [(2, 2, 1)]
    np.testing.assert_allclose(run.centres[:, 0], [12.0, 0.05, 0.3], rtol=1e-15)
    assert run.stop == "max_iter" and run.labels.tolist() == [1, 1, 2, 0]


def test_relocation_fills_empty_clusters_in_order_with_the_farthest_rows():
    x = np.array([[0.0], [1.0], [2.0], [10.0], [11.0], [30.0]])
    seeds = np.array([[100.0], [1.0], [90.0], [11.0], [95.0]])   # clusters 0, 2, 4 empty at the first assignment
    run = KO.lloyd(x, seeds, max_iter=1, tol_abs=0.0)
    assert run.iter_labels[0].tolist() == [1, 1, 1, 3, 3, 3]
    # distances to the old centres: 1, 0, 1, 1, 0, 361: row 5 first, then rows 0 and 2 (tie at 1: lowest row first),
    # row 3 (also at 1) stays
    assert run.relocations[0]["moves"] == [(0, 5, 3), (2, 0, 1), (4, 2, 1)]
    np.testing.assert_array_equal(run.centres[:, 0], [30.0, 1.0, 0.0, 10.5, 2.0])


def test_relocation_is_skipped_with_fewer_distinct_rows_than_clusters():
    base = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 2.0]])
    x = np.repeat(base, 4, axis=0)
    seeds = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 2.0], [0.0, 0.0], [1.0, 0.0]])   # duplicate seeds, k = 5 > 3
    run = KO.lloyd(x, seeds, max_iter=300, tol_abs=0.0)
    # every row sits on its centre: clusters 3 and 4 stay empty with their old centres, no row moves, and as no
    # centre moved the run stops on tol (0 <= 0) after one iteration; the shift is exact (the sums are)
    assert run.relocations[0]["moves"] == [] and run.relocations[0]["empty"] == [3, 4]
    assert run.stop == "tol" and run.n_iter == 1 and run.tol_margins == [math.inf]
    np.testing.assert_array_equal(run.centres, seeds)
    assert np.bincount(run.labels, minlength=5).tolist() == [4, 4, 4, 0, 0] and run.inertia == 0.0


def test_fit_picks_the_first_run_of_lowest_inertia():
    x = _blobs(300, 4, 5, seed=9, spread=1.0)
    f = KO.fit(x, 5, runs=6, seed=3, max_iter=300, tol_abs=0.0)
    inertia = f.inertia
    assert f.best == int(np.argmin(inertia)) and inertia[f.best] == inertia.min()
    for s, r in zip(f.seedings, f.runs):
        assert len(s.idx) == 5 and r.n_iter >= 1
    seeds_only = KO.fit(x, 5, runs=2, seed=3, max_iter=0, tol_abs=0.0)
    assert [r.n_iter for r in seeds_only.runs] == [0, 0]
    np.testing.assert_array_equal(seeds_only.runs[1].centres, x[f.seedings[1].idx])


def test_float32_centres_are_rounded_to_float32():
    x = _blobs(400, 6, 3, seed=4, spread=3.0).astype(np.float32)
    f = KO.fit(x, 3, runs=2, seed=1, max_iter=5, tol_abs=0.0)
    for r in f.runs:
        assert np.array_equal(r.centres.astype(np.float32).astype(np.float64), r.centres)
