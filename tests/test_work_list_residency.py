"""The resident-query filter keeps the query tile in shared memory across consecutive work items of one CTA with the
same q_row0.  Work lists contain such runs: a query tile whose train columns come in two ranges (stage 2: the
classes before and after its own) becomes two items, and one CTA's static share runs them back to back."""
import numpy as np

from simple_tip_b200 import engine as E


def _static_sequences(items, n_static, g):
    return [[tuple(items[i]) for i in range(b, n_static, g) if items[i][2] != items[i][3]] for b in range(g)]


def test_two_ranges_of_one_query_tile_run_back_to_back():
    tiles = [(r0, 128, [(0, 1024), (2048, 3072)], 1) for r0 in range(0, 512, 128)]
    items, n_static = E.build_balanced_items(tiles, 128, 2)
    g = min(2, len(items))
    runs = 0
    for seq in _static_sequences(items, n_static, g):
        runs += sum(1 for a, b in zip(seq, seq[1:]) if a[0] == b[0])
    assert runs > 0
    # every (query tile, train tile) pair is covered exactly once
    got = sorted((int(it[0]), c) for it in items for c in range(int(it[2]), int(it[3]), 128))
    want = sorted((r0, c) for r0, _, rng, _ in tiles for lo, hi in rng for c in range(lo, hi, 128))
    assert got == want
