"""The resident DSA filter on 192-row query tiles, bit for bit against the C oracle in both stages.

`pair_kernel<MODE_NN, *, RESA=true>` runs three consumer warpgroups, each on 64 rows of a 192-row query tile; one
whose rows all lie past the tile's last query issues no MMAs, hands the drain warps empty mailbox entries and keeps
its place in the ring.  Class-aligned query tiles end on a tile of (class size mod 192) rows, so class sizes of
384 + r put last tiles of r valid rows in both searches (stage 2's queries are stage 1's winners, with the same class
histogram).  A class whose training rows are all one row fills the event mailbox of every row of its tiles, rows
128-191 (the third warpgroup) included."""
import numpy as np
import pytest

from oracle import c_oracle

pytestmark = pytest.mark.gpu

TAILS = (1, 63, 64, 65, 128, 129, 191)


def _data(counts, n_train, d, seed, storm_classes=()):
    rng = np.random.default_rng(seed)
    classes = len(counts)
    centres = rng.normal(0.0, 2.0, size=(classes, d))
    ytr = rng.integers(0, classes, size=n_train)
    xtr = (centres[ytr] + rng.normal(size=(n_train, d))).astype(np.float32)
    for c in storm_classes:
        idx = np.flatnonzero(ytr == c)
        xtr[idx] = xtr[idx[0]]
    pte = rng.permutation(np.repeat(np.arange(classes), counts))
    xte = (centres[pte] + rng.normal(size=(len(pte), d))).astype(np.float32)
    return xtr, ytr.astype(np.int64), xte, pte.astype(np.int64)


def _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=3, pool_frac=0.5):
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import DSA

    monkeypatch.setattr(E, "POOL_FRAC", pool_frac)
    monkeypatch.setattr(E, "POOL_TILES", pool_tiles)
    monkeypatch.setattr(E, "POOL_MIN_TILES", 0)
    want = c_oracle.dsa(xtr, ytr, xte, pte)
    sa = DSA(xtr, ytr)
    assert sa._engine.resident and sa._engine.row_tile == 192
    for _ in range(3):          # eager launch, graph capture, graph replay
        got = sa(xte, pte)
        assert np.array_equal(got, want["dsa"])
        assert np.array_equal(sa.last_winner_index, want["idx_a"])
        assert np.array_equal(sa.last_dist_a, want["dist_a"]) and np.array_equal(sa.last_dist_b, want["dist_b"])


@pytest.mark.parametrize("d", [128, 48])
def test_last_tile_rows(monkeypatch, d):
    # one class per tail length: its last query tile holds 1 .. 191 valid rows, so 2, 1 or 0 warpgroups idle
    xtr, ytr, xte, pte = _data([384 + r for r in TAILS], 9000, d, seed=200 + d)
    _check(monkeypatch, xtr, ytr, xte, pte)


@pytest.mark.parametrize("storm", [0, 4, 6])
def test_event_storm_every_tile_row(monkeypatch, storm):
    # the storm class's training rows are one row: every chunk of its train tiles is an event for every query row of
    # its own tiles (stage 1) and for the queries whose nearest other class it is (stage 2), rows 0-191 alike
    xtr, ytr, xte, pte = _data([384 + r for r in TAILS], 8000, 128, seed=210 + storm, storm_classes=(storm,))
    _check(monkeypatch, xtr, ytr, xte, pte, pool_tiles=1 + storm % 3)


@pytest.mark.parametrize("classes", [12, 30])
def test_many_class_batch(monkeypatch, classes):
    # many classes of 384-575 queries: class-aligned tiles with every tail length, storms in every third class;
    # static work list only (no pool) for the 30-class case
    rng = np.random.default_rng(classes)
    counts = 384 + rng.integers(0, 192, size=classes)
    xtr, ytr, xte, pte = _data(counts, 12000, 128, seed=220 + classes, storm_classes=range(0, classes, 3))
    _check(monkeypatch, xtr, ytr, xte, pte, pool_frac=0.5 if classes == 12 else 0.0)
