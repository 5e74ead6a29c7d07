"""CPU tests of the float64 silhouette references (oracle/sil_oracle.py) that the device silhouette pass is compared
against: the references against sklearn, the packing emulation against its own spec, the finishing replica on
hand-built cases, and the power of the exact-case comparison: on the integer data of every layout the GPU tests use,
each kernel defect below is rejected."""
import numpy as np
import pytest

from oracle import sil_oracle as SO
from simple_tip_b200 import engine as E


def _sorted_case(x, labels):
    """label-sorted rows, encoded labels, counts and the sort order (what engine.silhouette_samples builds)"""
    _, codes = np.unique(labels, return_inverse=True)
    order = np.argsort(codes, kind="stable")
    counts = np.bincount(codes)
    return x[order], codes[order], counts, order


def _sklearn_cases():
    rng = np.random.default_rng(5)
    centres = rng.normal(size=(4, 6)) * 3.0
    lab = rng.integers(0, 4, size=300)
    blobs = centres[lab] + rng.normal(size=(300, 6))
    odd = np.where(lab == 2, 11, lab).astype(np.int64)      # arbitrary label values
    odd[7], odd[100] = -4, 99                                # two singleton clusters
    base = rng.integers(-6, 7, size=(30, 5)).astype(np.float64)
    dup = np.repeat(base, 8, axis=0)                          # every row 8 times; integer rows: exact distances
    dup_lab = np.repeat(rng.integers(0, 3, size=30), 8)
    return [("blobs", blobs, lab), ("label_values_and_singletons", blobs, odd), ("duplicates", dup, dup_lab),
            ("d1", rng.normal(size=(200, 1)), rng.integers(0, 3, size=200))]


@pytest.mark.parametrize("name", [c[0] for c in _sklearn_cases()])
def test_references_match_sklearn(name):
    from sklearn.metrics import silhouette_samples

    _, x, labels = next(c for c in _sklearn_cases() if c[0] == name)
    want = silhouette_samples(x, labels)
    assert np.max(np.abs(SO.exact_silhouette(x, labels) - want)) <= 1e-12
    # the same value from per-slot sums of the silhouette work list (2-tile spans)
    xs, lab_s, counts, order = _sorted_case(x, labels)
    items, slot_cluster = E.silhouette_items(counts, 2)
    part = SO.exact_dsum(xs, xs, items, slot_cluster.shape[0])
    assert not np.any(np.isnan(part))
    got = SO.silhouette_from_sums(SO.cluster_sums(part, slot_cluster, counts.shape[0]), lab_s, counts)
    assert np.max(np.abs(got - want[order])) <= 1e-12


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 15, 16, 17, 97])
def test_pack_sil_meets_its_spec(d, dtype):
    rng = np.random.default_rng(d)
    x = (rng.normal(size=(64, d)) * np.exp(rng.normal(size=(64, 1)) * 3)).astype(dtype)
    x[3] = 0.0
    center = rng.normal(size=d).astype(np.float32)
    q, t, nrm = SO.pack_sil(x, center)
    d16 = -(-d // 16) * 16
    assert q.shape == t.shape == (64, SO.pair_pitch(d)) and SO.pair_pitch(d) % 64 == 0
    val = lambda b: (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    qv, tv = val(q), val(t)
    v = (x.astype(np.float64) - center).astype(np.float32).astype(np.float64)
    h, lo = qv[:, :d], qv[:, d16:d16 + d]
    assert np.array_equal(qv[:, 2 * d16:2 * d16 + d], h)
    assert np.all(np.abs(v - (h + lo)) <= 2.0 ** -16 * np.abs(v))          # h + l = v to bf16^2 precision
    assert np.array_equal(tv[:, :d], -2 * h) and np.array_equal(tv[:, d16:d16 + d], -2 * h)
    assert np.array_equal(tv[:, 2 * d16:2 * d16 + d], -2 * lo)
    assert np.array_equal(nrm, np.sum(h * h + 2 * h * lo, axis=1).astype(np.float32))
    tail = tv[:, 3 * d16:3 * d16 + 3]
    assert np.array_equal(tail.sum(axis=1), nrm.astype(np.float64))        # the 3-way split sums back exactly
    assert np.all(qv[:, 3 * d16:3 * d16 + 3] == 1.0)
    for seg in range(3):                                                  # zero padding, d..d16 of every segment
        assert np.all(qv[:, seg * d16 + d:(seg + 1) * d16] == 0) and np.all(tv[:, seg * d16 + d:(seg + 1) * d16] == 0)
    assert np.all(qv[:, 3 * d16 + 3:] == 0) and np.all(tv[:, 3 * d16 + 3:] == 0)
    # the permutation selects rows
    perm = rng.permutation(64)
    qp, tp, np_ = SO.pack_sil(x, center, perm)
    assert np.array_equal(qp, q[perm]) and np.array_equal(tp, t[perm]) and np.array_equal(np_, nrm[perm])


def test_pack_sil_of_integer_rows_is_exact():
    rng = np.random.default_rng(1)
    x = rng.integers(-256, 257, size=(50, 40)).astype(np.float32)
    q, t, nrm = SO.pack_sil(x)
    val = lambda b: (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    qv, tv = val(q), val(t)
    assert np.array_equal(qv[:, :40], x) and not np.any(qv[:, 48:96]) and not np.any(tv[:, 96:144])
    assert np.array_equal(nrm.astype(np.float64), np.sum(x.astype(np.float64) ** 2, axis=1))
    assert np.array_equal(tv[:, 144:147].sum(axis=1), np.sum(x.astype(np.float64) ** 2, axis=1))


# ---- the exact case can see every defect -----------------------------------------------------------------------
LAYOUTS = SO.exact_layouts()


def _pair_dist(xq, xt, i, j):
    return np.sqrt(np.sum((xq[i] - xt[j]) ** 2, axis=-1))


def _spans(items):
    return sorted({(int(c0), int(c1), int(s)) for _, _, c0, c1, s, _ in items})


def _defects(x, y, items, ref):
    """(name, corrupted copy of ref) for each kernel defect; None when the defect changes nothing on this layout.
    An unwritten entry is modelled as 0 (production zero-fills part); NaN is rejected by the finiteness check."""
    n = x.shape[0]
    rows = np.arange(n)
    spans = _spans(items)
    own_slot = np.empty(n, dtype=np.int64)
    for c0, c1, s in spans:
        own_slot[c0:c1] = s
    out = []

    p = ref.copy()                                                       # no self mask
    p[own_slot, rows] += _pair_dist(x, y, rows, rows)
    out.append(("no_self_mask", p))
    for off in (-1, 1):                                                  # the mask on column i +- 1
        p = ref.copy()
        p[own_slot, rows] += _pair_dist(x, y, rows, rows)
        for c0, c1, s in spans:
            r = rows[(rows + off >= c0) & (rows + off < c1)]
            p[s, r] -= _pair_dist(x, y, r, r + off)
        out.append((f"mask_i{off:+d}", p))
    p = ref.copy()                                                       # last column of a partial tile dropped
    for c0, c1, s in spans:
        if (c1 - c0) % 128:
            r = rows[rows != c1 - 1]
            p[s, r] -= _pair_dist(x, y, r, np.full(r.shape, c1 - 1))
    out.append(("partial_tile_last_column_dropped", p))
    live = [sp for sp in spans if np.any(ref[sp[2]] > 0)]
    c0, c1, s = live[len(live) // 2]
    nb = s + 1 if s + 1 < ref.shape[0] else s - 1
    p = ref.copy()                                                       # one span written to a neighbouring slot
    p[nb], p[s] = ref[s], 0.0
    out.append(("span_in_neighbour_slot", p))
    p = ref.copy()                                                       # one span counted twice
    p[s] *= 2
    out.append(("span_counted_twice", p))
    p = ref.copy()                                                       # one (slot, row) entry left unwritten
    r = int(np.flatnonzero(ref[s] > 0)[0])
    p[s, r] = 0.0
    out.append(("entry_unwritten", p))
    return [(name, None if np.array_equal(p, ref) else p) for name, p in out]


@pytest.mark.parametrize("layout", LAYOUTS, ids=[lay[0] for lay in LAYOUTS])
def test_exact_case_detects_every_defect(layout):
    name, counts, d, _ = layout
    x, y = SO.layout_operands(layout)
    assert np.array_equal(x, np.round(x)) and np.abs(x).max() <= SO.INT_RANGE
    off = np.concatenate([[0], np.cumsum(counts)])
    # detectability: inside every cluster (so inside any span of it) each other column's distance and the row's own
    # column distance exceed 4 * beta * (the row's sum over the whole cluster), which bounds every span's sum
    for c0, c1 in zip(off[:-1], off[1:]):
        for r0 in range(c0, c1, 2048):
            r1 = min(c1, r0 + 2048)
            dist = np.sqrt(np.maximum(np.sum(x[r0:r1] ** 2, 1)[:, None] + np.sum(y[c0:c1] ** 2, 1)[None]
                                      - 2 * x[r0:r1] @ y[c0:c1].T, 0))
            rr = np.arange(r1 - r0)
            own = dist[rr, rr + r0 - c0].copy()
            dist[rr, rr + r0 - c0] = np.inf
            total = np.where(np.isinf(dist), 0, dist).sum(1)
            thr = 4 * SO.dsum_bound(total)
            assert np.all(own > thr) and np.all(own >= SO.INT_SHIFT)
            assert np.all(dist.min(1, initial=np.inf) > thr), name
    applied = set()
    for span_tiles in (1, 2, 16):
        items, slot_cluster = E.silhouette_items(np.asarray(counts), span_tiles)
        SO.check_work_list(items, slot_cluster, counts, span_tiles)
        ref = SO.exact_dsum(x, y, items, slot_cluster.shape[0])
        assert not np.any(np.isnan(ref)) and SO.dsum_excess(ref, ref) == 0.0
        noisy = ref * (1 + 0.9 * SO.BETA * np.cos(np.arange(ref.size)).reshape(ref.shape))
        assert SO.dsum_excess(noisy.astype(np.float32), ref) <= 1.0         # float32 storage inside the budget
        for defect, bad in _defects(x, y, items, ref):
            if bad is None:
                continue
            applied.add(defect)
            # the device's own error (<= beta * ref) cannot hide the defect either
            assert SO.dsum_excess(bad, ref) > 4.0, (name, span_tiles, defect)
            nan = bad.copy()
            nan[bad != ref] = np.nan
            assert SO.dsum_excess(nan, ref) == np.inf
    must = {"no_self_mask", "span_in_neighbour_slot", "span_counted_twice", "entry_unwritten", "mask_i+1"}
    assert must <= applied, (name, must - applied)


def test_every_defect_applies_somewhere():
    """some defects change nothing on some layouts (dropping the last column of a partial tile, when every partial
    span is a singleton's own column); across the layout matrix every defect is exercised"""
    applied = set()
    for layout in LAYOUTS:
        if sum(layout[1]) > 5000:
            continue
        x, y = SO.layout_operands(layout)
        items, slot_cluster = E.silhouette_items(np.asarray(layout[1]), 1)
        ref = SO.exact_dsum(x, y, items, slot_cluster.shape[0])
        applied |= {name for name, bad in _defects(x, y, items, ref) if bad is not None}
    assert applied == {"no_self_mask", "mask_i-1", "mask_i+1", "partial_tile_last_column_dropped",
                       "span_in_neighbour_slot", "span_counted_twice", "entry_unwritten"}


def test_check_work_list_rejects_broken_lists():
    counts = np.array([300, 1, 0, 700])
    items, slot_cluster = E.silhouette_items(counts, 1)
    SO.check_work_list(items, slot_cluster, counts, 1)
    with pytest.raises(AssertionError):
        SO.check_work_list(items, slot_cluster, counts, 1, col_tile=128)      # spans wider than allowed

    def broken(edit):
        it, sc = items.copy(), slot_cluster.copy()
        edit(it, sc)
        with pytest.raises(AssertionError):
            SO.check_work_list(it, sc, counts, 1)

    last = lambda it: np.flatnonzero(it[:, 4] == it[:, 4].max())
    broken(lambda it, sc: it.__setitem__((0, 3), it[0, 3] - 1))                # a column of a span dropped
    broken(lambda it, sc: it.__setitem__((last(it), 2), it[last(it), 2] - 1))  # spans overlap
    broken(lambda it, sc: it.__setitem__((0, 1), it[0, 1] - 1))                # a query row missing from a slot
    broken(lambda it, sc: it.__setitem__((1, 0), it[0, 0]))                    # a query tile twice, another missing
    broken(lambda it, sc: sc.__setitem__(1, sc[0] + 2))                        # a slot in the wrong cluster
    broken(lambda it, sc: it.__setitem__((0, 4), it[0, 4] + 1))                # an item in the neighbouring slot


# ---- the finishing replica -------------------------------------------------------------------------------------
def test_finish_replica_hand_built_cases():
    # clusters: 0 = rows {0, 1, 2}, 1 = row {3} (singleton), 2 = rows {4, 5}; one slot per cluster
    lab = np.array([0, 0, 0, 1, 2, 2])
    counts = np.array([3, 1, 2])
    part = np.array([[2.0, 4.0, 6.0, 9.0, 30.0, 30.0],      # sums to cluster 0
                     [8.0, 8.0, 8.0, 0.0, 12.0, 1.0],       # sums to cluster 1
                     [10.0, 12.0, 14.0, 5.0, 4.0, 4.0]],    # sums to cluster 2
                    dtype=np.float32)
    got = SO.finish_replica(part, np.array([0, 1, 2]), lab, counts, None)
    # row 0: a = 2 / 2 = 1, b = min(8 / 1, 10 / 2) = 5 -> 0.8; row 3: singleton -> 0
    assert got[0] == (5.0 - 1.0) / 5.0 and got[3] == 0.0
    # row 5: a = 4 / 1 = 4, b = min(30 / 3, 1 / 1) = 1 < a -> (1 - 4) / 4
    assert got[5] == (1.0 - 4.0) / 4.0
    # a = b = 0 -> 0 (sklearn's nan_to_num), not NaN
    z = np.zeros((3, 6), dtype=np.float32)
    assert np.array_equal(SO.finish_replica(z, np.array([0, 1, 2]), lab, counts, None), np.zeros(6))
    # a single cluster present: b stays +inf -> 0
    one = SO.finish_replica(np.ones((2, 4), dtype=np.float32), np.array([0, 0]), np.zeros(4, dtype=int),
                            np.array([4]), None)
    assert np.array_equal(one, np.zeros(4))
    # slots merge per cluster in ascending order, out_idx scatters
    part2 = np.concatenate([part[:1] / 2, part[:1] / 2, part[1:]]).astype(np.float32)
    perm = np.array([5, 0, 4, 1, 3, 2])
    got2 = SO.finish_replica(part2, np.array([0, 0, 1, 2]), lab, counts, perm)
    assert np.array_equal(got2[perm], got)


def test_finish_replica_agrees_with_the_sklearn_formula():
    rng = np.random.default_rng(3)
    counts = np.array([1, 40, 7, 2, 90])
    lab = np.repeat(np.arange(5), counts)
    slot_cluster = np.repeat(np.arange(5), [1, 3, 1, 2, 4])
    part = rng.uniform(0.5, 100.0, size=(slot_cluster.shape[0], lab.shape[0])).astype(np.float32)
    got = SO.finish_replica(part, slot_cluster, lab, counts, None)
    want = SO.silhouette_from_sums(SO.cluster_sums(part, slot_cluster, 5), lab, counts)
    assert np.max(np.abs(got - want)) <= 1e-15 and np.all(got[lab == 0] == 0.0)
