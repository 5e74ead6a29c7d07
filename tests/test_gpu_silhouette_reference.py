"""GPU tests of the silhouette pass (tip_sil_prep -> tip_sil_dsum -> tip_sil_finish) against float64 references of
its own operands (oracle/sil_oracle.py), through the C ABI:

  * the packing bit for bit (sqnorm to 1 fp32 ulp: the device's double warp sum may order terms differently);
  * the per-(slot, row) distance sums on integer rows, where every operand, product and partial sum is exact and the
    device's only errors are sqrt.approx and fp32 summation: within beta = 1e-6 of the exact sum, own column masked,
    every slot written (part is NaN-filled first); 1-, 2- and 16-tile spans and the card's own choice;
  * tip_sil_finish bit for bit against a NumPy replica of its double arithmetic;
  * the whole pass end to end against the float64 silhouette of the input at DESIGN.md §4b's tolerances, and the
    best k of a model selection.
Lines starting with [sil-ref] report the worst errors (run with -s to see them)."""
import math

import numpy as np
import pytest

from oracle import sil_oracle as SO

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64


def _env():
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    return torch, _lib, _lib.load(), E


def _prep(xd, center=None, src_idx=None):
    """tip_sil_prep of the rows src_idx (None: all) of the device matrix xd -> (q_pack, t_pack, sqnorm); the outputs
    start as a NaN bit pattern, so a column the kernel never writes cannot pass for a zero"""
    torch, _lib, lib, E = _env()
    n, d = xd.shape
    rows = n if src_idx is None else src_idx.shape[0]
    pitch = int(lib.tip_pair_pitch(d, 3))
    q = torch.full((rows, pitch), 0x7FC1, dtype=torch.int16, device=xd.device).view(torch.bfloat16)
    t = torch.full((rows, pitch), 0x7FC1, dtype=torch.int16, device=xd.device).view(torch.bfloat16)
    sq = torch.full((rows,), float("nan"), dtype=torch.float32, device=xd.device)
    _lib.check(lib.tip_sil_prep(E._p(xd), E.tip_dtype(xd.dtype), rows, d, E._p(center), E._p(src_idx), E._p(q), E._p(t),
                                E._p(sq), E._stream()), "tip_sil_prep")
    return q, t, sq


def _bits(p):
    return p.view(_env()[0].int16).cpu().numpy().view(np.uint16)


# ---- packing ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [f32, f64])
@pytest.mark.parametrize("d", [1, 15, 16, 17, 96, 97, 2048])
def test_sil_prep_packs_bit_for_bit(d, dtype):
    torch = _env()[0]
    rng = np.random.default_rng(d * 2 + (dtype == f64))
    n = 300
    x = (rng.normal(size=(n, d)) * np.exp(rng.normal(size=(n, 1)) * 2.0)).astype(dtype)
    center = (rng.normal(size=d) * 0.5).astype(f32)
    x[5], x[6], x[7] = 0.0, -0.0, center                 # zero rows and a row on the centre (v = 0)
    x[8] = np.round(x[8] * 8) / 8                         # bf16-exact values: l = 0
    xd = torch.from_numpy(x).cuda()
    perm = rng.permutation(n).astype(np.int32)
    d16 = -(-d // 16) * 16
    tail = np.zeros(SO.pair_pitch(d), dtype=bool)
    tail[3 * d16:3 * d16 + 3] = True
    for cen in (None, center):
        for order in (None, perm):
            q, t, sq = _prep(xd, None if cen is None else torch.from_numpy(cen).cuda(),
                             None if order is None else torch.from_numpy(order).cuda())
            wq, wt, wsq = SO.pack_sil(x, cen, order)
            dq, dt, dsq = _bits(q), _bits(t), sq.cpu().numpy()
            where = f"d={d} {np.dtype(dtype).name} center={cen is not None} perm={order is not None}"
            assert np.array_equal(dq, wq), (where, np.argwhere(dq != wq)[:4].tolist())
            assert np.array_equal(dt[:, ~tail], wt[:, ~tail]), (where, np.argwhere(dt[:, ~tail] != wt[:, ~tail])[:4].tolist())
            assert np.all(np.abs(dsq - wsq) <= np.spacing(wsq)), (where, float(np.max(np.abs(dsq - wsq) / np.spacing(wsq))))
            # the norm term is the 3-way split of the norm the kernel reports
            assert np.array_equal(dt[:, tail], SO.bf16_bits(SO.split3(dsq))), where


# ---- exact distance sums ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 16, 96, 97, 300, 2048])
def test_integer_operands_accumulate_exactly(d):
    """the premise of the exact case: on these operands the tensor-core K-loop yields T(y_j) - 2<x_i, y_j> exactly,
    in the resident-query kernel (d <= 96) and in the streaming one"""
    torch, _lib, lib, E = _env()
    x, y = SO.int_operands([256], d, seed=d)
    qx, _, sqx = _prep(torch.from_numpy(x.astype(f32)).cuda())
    _, ty, sqy = _prep(torch.from_numpy(y.astype(f32)).cuda())
    assert np.array_equal(sqx.cpu().numpy(), np.sum(x * x, 1)) and np.array_equal(sqy.cpu().numpy(), np.sum(y * y, 1))
    want = np.sum(y * y, 1)[None, :] - 2.0 * x[:128] @ y.T
    pitch = int(lib.tip_pair_pitch(d, 3))
    for variant in ((1, 2) if d <= 96 else (1,)):
        out = torch.full((256, 256), float("nan"), dtype=torch.float32, device="cuda")
        _lib.check(lib.tip_pair_probe(E._p(qx), 256, E._p(ty), 256, d, 3, pitch, variant, E._p(out), E._stream()),
                   "tip_pair_probe")
        got = out[:128].cpu().numpy().astype(f64)
        assert np.array_equal(got, want), (d, variant, float(np.nanmax(np.abs(got - want))))


def _dsum(qx, ty, sqx, n, d, items, slots):
    torch, _lib, lib, E = _env()
    part = torch.full((slots, n), float("nan"), dtype=torch.float32, device="cuda")
    items_dev = torch.from_numpy(np.ascontiguousarray(items)).cuda()
    _lib.check(lib.tip_sil_dsum(E._p(qx), E._p(ty), E._p(sqx), n, d, int(lib.tip_pair_pitch(d, 3)), E._p(items_dev),
                                items.shape[0], E._p(part), E._stream()), "tip_sil_dsum")
    return part.cpu().numpy()


LAYOUTS = SO.exact_layouts()


@pytest.mark.parametrize("layout", LAYOUTS, ids=[lay[0] for lay in LAYOUTS])
def test_sil_dsum_matches_exact_sums(layout):
    torch, _lib, lib, E = _env()
    name, counts, d, _ = layout
    x, y = SO.layout_operands(layout)
    n = x.shape[0]
    qx, _, sqx = _prep(torch.from_numpy(x.astype(f32)).cuda())
    _, ty, _ = _prep(torch.from_numpy(y.astype(f32)).cuda())
    pairs = math.ceil(n / _lib.ROW_TILE) * math.ceil(n / _lib.COL_TILE)
    choices = sorted({1, 2, 16, E.span_tiles_for(pairs, E._device_sms(lib))})
    worst = []
    for span_tiles in choices:
        items, slot_cluster = E.silhouette_items(np.asarray(counts), span_tiles)
        SO.check_work_list(items, slot_cluster, counts, span_tiles)   # the reference below follows the list it is given
        slots = slot_cluster.shape[0]
        part = _dsum(qx, ty, sqx, n, d, items, slots)
        ref = SO.exact_dsum(x, y, items, slots, device="cuda")
        assert not np.any(np.isnan(ref))
        assert np.all(np.isfinite(part)), (name, span_tiles, "unwritten (slot, row) entries",
                                           np.argwhere(~np.isfinite(part))[:4].tolist())
        excess = SO.dsum_excess(part, ref)
        assert excess <= 1.0, (name, span_tiles, excess)
        worst.append(excess)
    print(f"[sil-ref] exact sums {name} (n={n}, d={d}, {len(counts)} clusters): worst |err| / bound "
          f"{max(worst):.3g} over span_tiles {choices}")


# ---- the finishing kernel --------------------------------------------------------------------------------------
def _finish_case(n, n_clusters, seed, one_cluster=False):
    rng = np.random.default_rng(seed)
    if one_cluster:
        counts = np.zeros(n_clusters, dtype=np.int64)
        counts[0] = n
    else:
        counts = np.bincount(rng.integers(0, n_clusters, size=n), minlength=n_clusters)
        for c in range(0, n_clusters, 7):                # a few singleton clusters
            if counts[c] >= 1:
                counts[(c + 1) % n_clusters] += counts[c] - 1
                counts[c] = 1
    lab = np.repeat(np.arange(n_clusters), counts).astype(np.int32)
    slot_cluster = np.repeat(np.arange(n_clusters), rng.integers(1, 4 if n_clusters <= 64 else 3,
                                                                 size=n_clusters)).astype(np.int32)
    if one_cluster:
        slot_cluster = np.zeros(3, dtype=np.int32)
    part = rng.uniform(0.01, 1000.0, size=(slot_cluster.shape[0], n)).astype(f32)
    part[:, rng.integers(0, n, size=max(1, n // 50))] = 0.0      # rows with a = b = 0
    return part, slot_cluster, lab, counts.astype(np.int32)


FINISH = [(n, c, False) for n in (1, 255, 256, 257, 100_000) for c in (2, 64, 500)] + [(257, 2, True)]


@pytest.mark.parametrize("n, n_clusters, one_cluster", FINISH)
def test_sil_finish_is_bit_exact(n, n_clusters, one_cluster):
    torch, _lib, lib, E = _env()
    part, slot_cluster, lab, counts = _finish_case(n, n_clusters, seed=n + n_clusters, one_cluster=one_cluster)
    perm = np.random.default_rng(n).permutation(n).astype(np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    part_d, sc_d, lab_d, cnt_d = dev(part), dev(slot_cluster), dev(lab), dev(counts)
    for out_idx in (None, perm):
        out = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        _lib.check(lib.tip_sil_finish(E._p(part_d), n, slot_cluster.shape[0], E._p(sc_d), E._p(lab_d), E._p(cnt_d),
                                      E._p(None if out_idx is None else dev(out_idx)), E._p(out), E._stream()),
                   "tip_sil_finish")
        got = out.cpu().numpy()
        want = SO.finish_replica(part, slot_cluster, lab, counts, out_idx)
        bad = np.flatnonzero(got.view(np.int64) != want.view(np.int64))
        assert bad.size == 0, (n, n_clusters, out_idx is not None, int(bad[0]), got[bad[0]], want[bad[0]])
    print(f"[sil-ref] finish n={n} clusters={n_clusters}{' (one present)' if one_cluster else ''}: bit-exact")


# ---- end to end on real-valued data ----------------------------------------------------------------------------
def _e2e_data(counts, d, dtype, seed, offset=0.0):
    """rows of cluster c around their own centre, shuffled: labels as k-means would hand them over"""
    rng = np.random.default_rng(seed)
    k = len(counts)
    centres = rng.normal(size=(k, d)) * (3.0 if d > 1 else 6.0)
    lab = np.repeat(np.arange(k), counts)
    x = centres[lab] + rng.normal(size=(lab.shape[0], d))
    perm = rng.permutation(lab.shape[0])
    return (x[perm] + offset).astype(dtype), lab[perm] * 3 - 5           # arbitrary label values


_SIZES = LAYOUTS[0][1]
_C64 = LAYOUTS[2][1]
_C500 = LAYOUTS[4][1]
# name, cluster sizes, d, dtype, offset, tolerance regime (DESIGN.md §4b):
#   "tol"          1e-4 per row (5e-4 for d = 1) and 1e-5 on the score;
#   "small_d1"     d = 1, 16 or 500 overlapping clusters, small ones among them, rows up to 15 spreads from the centre:
#                  every row is held to the worst-case bound of the §4b error model for its own data.  Measured there:
#                  0.015 / 0.067 per row, and 8.0e-4 even on rows whose a and every possible b average over >= 128
#                  rows (DESIGN.md §4b: pairs closer than a bf16 step 2^-8 |x| lose their distance);
#   "biased_score" the one shape measured with a score error above 1e-5 (rows at 1e-4, score at the row tolerance)
E2E = [
    ("sizes_d97_f32", _SIZES, 97, f32, 0.0, "tol"),
    ("sizes_d1_f64", _SIZES, 1, f64, 0.0, "small_d1"),
    ("c64_d2048_f32", _C64, 2048, f32, 0.0, "biased_score"),
    ("c64_d97_f64", _C64, 97, f64, 0.0, "tol"),
    ("c500_d1_f32", _C500, 1, f32, 0.0, "small_d1"),
    ("n129_128_1_d2048_f64", [128, 1], 2048, f64, 0.0, "tol"),
    ("n129_1_128_d97_f32", [1, 128], 97, f32, 0.0, "tol"),
    ("n4097_d2048_f32", [2049, 2048], 2048, f32, 0.0, "tol"),
    ("n20000_d97_f32", [12000, 8000], 97, f32, 0.0, "tol"),
    ("n20000_d1_f64", [12000, 8000], 1, f64, 0.0, "tol"),
    ("c64_d97_offset_f64", _C64, 97, f64, 1e4, "tol"),
]


@pytest.mark.parametrize("case", E2E, ids=[c[0] for c in E2E])
def test_silhouette_end_to_end_matches_exact(case):
    torch, _lib, lib, E = _env()
    from simple_tip_b200.core import clustering

    name, counts, d, dtype, offset, regime = case
    x, labels = _e2e_data(counts, d, dtype, seed=len(counts) * 13 + d, offset=offset)
    want = SO.exact_silhouette(x, labels, device="cuda")
    row_tol = np.full(x.shape[0], 5e-4 if d == 1 else 1e-4)
    score_tol = 1e-5
    averaged = np.ones(x.shape[0], dtype=bool)
    if regime == "small_d1":
        # near pairs in one dimension are pure cancellation, and a mean over a few rows averages nothing away
        bound, support = SO.silhouette_error_bound(x, labels, device="cuda")
        averaged = support >= 128            # reported: the rows a fixed 5e-4 was measured for on other data
        row_tol = bound + 1e-7
        # no bound on the score beyond what the row checks imply: |mean error| <= mean of the row limits
        score_tol = float(np.mean(row_tol))
    elif regime == "biased_score":
        # measured: the row errors share one sign, so their mean does not shrink; the score is held to the row
        # tolerance, which the row check already implies
        score_tol = 1e-4
    got = clustering.silhouette_samples(x, labels)
    score = clustering.silhouette_score(x, labels)
    results = {"default": got}
    _, codes = np.unique(labels, return_inverse=True)
    xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(codes).cuda()
    for span_tiles in (1, 16):
        results[f"span_tiles={span_tiles}"] = E.silhouette_samples(xd, cd, len(counts), span_tiles=span_tiles).cpu().numpy()
    errs = {k: float(np.max(np.abs(v - want))) for k, v in results.items()}
    over = {k: float(np.max(np.abs(v - want) / row_tol)) for k, v in results.items()}
    score_err = abs(score - float(np.mean(want)))
    dev = got - want
    print(f"[sil-ref] end to end {name} (n={x.shape[0]}, {regime}): max row err {max(errs.values()):.3g} "
          f"(max err / tol {max(over.values()):.3g}, tol {np.min(row_tol):.3g}..{np.max(row_tol):.3g}), "
          f"score err {score_err:.3g} (tol {score_tol:.3g}); averaged rows {int(averaged.sum())}/{x.shape[0]} with max "
          f"err {float(np.max(np.abs(dev[averaged]), initial=0.0)):.3g} "
          f"(err / tol {float(np.max(np.abs(dev[averaged]) / row_tol[averaged], initial=0.0)):.3g}); "
          f"rows with err > 0: {float(np.mean(dev > 0)):.2f}; "
          f"{errs}")
    assert all(o <= 1.0 for o in over.values()), (name, over)
    assert score_err <= score_tol, (name, score_err)


@pytest.mark.parametrize("d", [32, 200])
def test_silhouette_end_to_end_with_heavy_duplication(d):
    from simple_tip_b200.core import clustering

    rng = np.random.default_rng(d)
    centres = rng.normal(size=(3, d)) * 2.0
    lab = rng.integers(0, 3, size=60)
    base = (centres[lab] + rng.normal(size=(60, d))).astype(f32)
    x, labels = np.repeat(base, 25, axis=0), np.repeat(lab, 25)
    want = SO.exact_silhouette(x, labels, device="cuda")
    row_err = float(np.max(np.abs(clustering.silhouette_samples(x, labels) - want)))
    score_err = abs(clustering.silhouette_score(x, labels) - float(np.mean(want)))
    print(f"[sil-ref] end to end duplicates d={d}: max row err {row_err:.3g} (tol 5e-4), score err {score_err:.3g} "
          f"(tol 2e-4)")
    assert row_err <= 5e-4 and score_err <= 2e-4


def test_model_selection_picks_the_exact_best_k():
    """for each candidate k: the device's k-means labels, scored by the device silhouette and by the float64 one; the
    device must pick the exact best k whenever the exact scores leave it clear of twice the score tolerance"""
    from simple_tip_b200.core.clustering import KMeans, silhouette_score

    rng = np.random.RandomState(42)      # the reference's k-means MultiModalSA test data
    mmdsa = np.concatenate([rng.random((100, 10)), rng.random((100, 10)) + 0.9])
    g = np.random.default_rng(8)
    centres = g.normal(size=(5, 24)) * 3.0
    blobs = centres[g.integers(0, 5, size=3000)] + g.normal(size=(3000, 24))
    for name, x, ks in (("mmdsa", mmdsa, [2, 3, 4]), ("blobs", blobs, list(range(2, 9)))):
        dev, ex = [], []
        for k in ks:
            lab = KMeans(k, n_init=10, random_state=0).fit(x).labels_
            dev.append(silhouette_score(x, lab))
            ex.append(float(np.mean(SO.exact_silhouette(x, lab, device="cuda"))))
        dev, ex = np.array(dev), np.array(ex)
        assert np.max(np.abs(dev - ex)) <= 1e-5, (name, dev, ex)
        top = np.argsort(ex)[::-1]
        clear = ex[top[0]] - ex[top[1]] > 2e-5
        if clear:
            assert int(np.argmax(dev)) == top[0], (name, dev, ex)
        print(f"[sil-ref] model selection {name}: best k exact {ks[top[0]]}, device {ks[int(np.argmax(dev))]}, "
              f"gap {ex[top[0]] - ex[top[1]]:.3g}, max score err {np.max(np.abs(dev - ex)):.3g}")
