"""The DSA filter's event path at its worst case, bit for bit against the C oracle.

The consumer warps of the filter (`pair_kernel<MODE_NN>`) record each chunk whose minimum lies inside its row's window
in a per-tile mailbox; the drain warps stage, compact and emit them.  These cases fill the mailbox: a class whose
training rows are all identical (every chunk of every tile is an event for every row), exact ties placed on both
sides of a train-tile boundary, pool items of 1-3 tiles, and many-class batches, where the other-class search
excludes each query's own class."""
import numpy as np
import pytest

from oracle import c_oracle, np_oracle

pytestmark = pytest.mark.gpu


def _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=4, pool_frac=0.5):
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import DSA

    monkeypatch.setattr(E, "POOL_FRAC", pool_frac)
    monkeypatch.setattr(E, "POOL_TILES", pool_tiles)
    monkeypatch.setattr(E, "POOL_MIN_TILES", 0)
    want = c_oracle.dsa(xtr, ytr, xte, pte)
    sa = DSA(xtr, ytr)
    for _ in range(3):          # eager launch, graph capture, graph replay
        got = sa(xte, pte)
        assert np.array_equal(got, want["dsa"])
        assert np.array_equal(sa.last_winner_index, want["idx_a"])
        assert np.array_equal(sa.last_dist_a, want["dist_a"]) and np.array_equal(sa.last_dist_b, want["dist_b"])


@pytest.mark.parametrize("pool_tiles", [1, 2, 3])
def test_identical_class_saturates_events(monkeypatch, pool_tiles):
    # class 0's 1000 training rows are one row: every value of every tile ties, so every chunk is an event
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(4000, 600, 128, 4, seed=70 + pool_tiles)
    xtr[ytr == 0] = xtr[np.flatnonzero(ytr == 0)[0]]
    _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=pool_tiles)


def test_near_ties_across_tile_boundaries(monkeypatch):
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(6000, 800, 128, 3, seed=81)
    order = np.argsort(ytr, kind="stable")
    xtr, ytr = xtr[order], ytr[order]
    rng = np.random.default_rng(5)
    # queries sit on training rows that straddle 128-row boundaries; their twins on the other side differ in one ulp
    for k, j in enumerate(range(127, len(xtr) - 1, 128)):
        if ytr[j] != ytr[j + 1] or k >= len(xte):
            continue
        xtr[j + 1] = np.nextafter(xtr[j], np.float32(np.inf)) if k % 2 else xtr[j]
        xte[k] = xtr[j] + rng.normal(scale=1e-3, size=xtr.shape[1]).astype(np.float32)
        pte[k] = ytr[j]
    _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=2)


@pytest.mark.parametrize("classes", [10, 23])
def test_many_class_batches_excluded_ranges(monkeypatch, classes):
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(9000, 2000, 128, classes, seed=90 + classes)
    # every other class gets a block of identical rows, so the excluded and included ranges both carry event storms
    for c in range(0, classes, 2):
        idx = np.flatnonzero(ytr == c)[:200]
        xtr[idx] = xtr[idx[0]]
    _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=3)
