"""CPU tests: host-side planning, the C-ABI export table, and the cross-rank protocol
(world_size-2 gloo).  No compute call touches a GPU here."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import np_oracle
from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def test_c_abi_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "b200tip.h")).read()
    declared = set(re.findall(r"\b(tip_[a-z0-9_]+)\s*\(", header))
    declared -= {"tip_status", "tip_dtype", "tip_work_item", "tip_comm"}
    assert declared == set(_lib.symbols()), declared ^ set(_lib.symbols())
    lib = _lib.load()                      # static cudart: loads without a GPU
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.tip_version() == 200
    assert lib.tip_pair_pitch(128, 1) == 192 and lib.tip_pair_pitch(256, 3) == 832
    assert lib.tip_pair_pitch(5, 1) == 64 and lib.tip_pair_pitch(0, 1) == -1
    assert C.sizeof(_lib.WorkItem) == 24
    assert C.sizeof(_lib.RerankExtras) == 72 == lib.tip_sizeof_rerank_extras()


def test_ctypes_signatures_have_the_header_arity():
    """Every prototype of include/b200tip.h and its ctypes binding take the same number of arguments
    (a mismatch would corrupt the call silently)."""
    header = open(os.path.join(ROOT, "include", "b200tip.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = dict(re.findall(r"\b(tip_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", header, flags=re.S))
    assert set(protos) == set(_lib.symbols())
    for name, params in protos.items():
        params = params.strip()
        n_header = 0 if params in ("", "void") else params.count(",") + 1
        assert n_header == len(_lib._SIGNATURES[name][1]), (name, n_header, len(_lib._SIGNATURES[name][1]))


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "simple_tip_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in text.lower().replace("# oracle", ""), f"{f} mentions the oracle"


def test_scoring_fails_loudly_without_a_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from src.core.deepgini import DeepGini
    from src.core.surprise import DSA

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DeepGini.calculate(np.ones((2, 2), dtype=np.float32) / 2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DSA(np.zeros((4, 3), dtype=np.float32), np.array([0, 1, 0, 1]))


def test_class_layout_and_subsampling_match_reference_semantics(golden):
    labels = np.array([2, 0, 1, 2, 5, 0, 1, 1, -1, 2])
    order, off = E.class_layout(labels, 3)
    assert list(off) == [0, 2, 5, 8]
    assert list(order) == [1, 5, 2, 6, 7, 0, 3, 9]          # ascending position inside each class
    # sub-sampling picks the same rows as the reference (surprise.py:84-86)
    from src.core.surprise import _subsample_arrays

    a = np.arange(1000)
    (got,) = _subsample_arrays(0.3, (a,), seed=0)
    want = np_oracle.subsample_indexes(1000, 0.3, 0)
    assert np.array_equal(got, want) and got.shape == (300,)
    (got,) = _subsample_arrays(17, (a,), seed=3)
    assert np.array_equal(got, np.random.RandomState(3).choice(np.arange(1000), 17, replace=False))
    assert _subsample_arrays(1.0, (a,), seed=0)[0] is a
    with pytest.raises(ValueError):
        _subsample_arrays(0, (a,), seed=0)


def test_work_items_cover_every_pair_exactly_once():
    rng = np.random.default_rng(0)
    q_off = np.array([0, 300, 300, 1000])                    # class 1 has no queries
    t_off = np.array([0, 5000, 5600, 9000])
    for mode in ("same", "other"):
        ranges = [[(t_off[c], t_off[c + 1])] if mode == "same" else [(0, t_off[c]), (t_off[c + 1], t_off[-1])]
                  for c in range(3)]
        items, slots = E.build_items(q_off, ranges, span_tiles=3)
        cover = np.zeros((1000, 9000), dtype=np.int32)
        for q0, rows, c0, c1, slot, _ in items:
            assert 1 <= rows <= 128 and c1 - c0 <= 3 * 256 and 0 <= slot < slots
            cover[q0:q0 + rows, c0:c1] += 1
        want = np.zeros_like(cover)
        for c in range(3):
            for lo, hi in ranges[c]:
                want[q_off[c]:q_off[c + 1], lo:hi] = 1
        assert np.array_equal(cover, want)
        assert E.count_tile_pairs(q_off, ranges) >= items.shape[0]
    assert E.build_items(np.array([0, 0]), [[(0, 10)]], 2)[0].shape == (0, 6)
    assert 2 <= E.span_tiles_for(10, 148) <= 16 and E.span_tiles_for(10 ** 7, 148) == 16
    # span-major order: the same items, sorted by (train span, query tile)
    sm = E.span_major(items)
    assert sorted(map(tuple, sm.tolist())) == sorted(map(tuple, items.tolist()))
    assert np.all(np.diff(sm[:, 2]) >= 0)


def test_other_class_items_cover_every_pair_exactly_once():
    """Stage-2 work list: tiles ignore class boundaries; single-class tiles skip their own class's
    train rows, mixed tiles scan everything and rely on the per-query mask (flag bit 0)."""
    for q_off, t_off in [(np.array([0, 300, 300, 1000]), np.array([0, 5000, 5600, 9000])),
                         (np.arange(0, 1001, 10), np.arange(0, 16001, 160)),          # 100 classes of 10 queries
                         (np.array([0, 7]), np.array([0, 50]))]:
        m, n = int(q_off[-1]), int(t_off[-1])
        classes = len(q_off) - 1
        q_class = np.repeat(np.arange(classes), np.diff(q_off))
        for row_tile, col_tile in ((128, 256), (256, 128)):
            items = E.build_other_class_items(q_off, t_off, row_tile, col_tile, lambda pairs: 3)
            cover = np.zeros((m, n), dtype=np.int32)
            for q0, rows, c0, c1, slot, flag in items:
                assert 1 <= rows <= row_tile and 0 < c1 - c0 <= 3 * col_tile
                block = np.ones((rows, c1 - c0), dtype=np.int32)
                if flag & 1:      # the kernel masks each query's own class
                    for r in range(rows):
                        c = q_class[q0 + r]
                        lo, hi = max(t_off[c], c0), min(t_off[c + 1], c1)
                        if hi > lo:
                            block[r, lo - c0:hi - c0] = 0
                else:
                    assert len(set(q_class[q0:q0 + rows])) == 1
                cover[q0:q0 + rows, c0:c1] += block
            want = np.ones((m, n), dtype=np.int32)
            for c in range(classes):
                want[q_off[c]:q_off[c + 1], t_off[c]:t_off[c + 1]] = 0
            assert np.array_equal(cover, want)


def test_balanced_items_cover_every_pair_once_and_balance_the_static_schedule():
    """Work list of the resident-query kernel: equal train-tile counts per CTA under the kernel's
    `item = CTA + round * G` schedule for the static items (padding entries, col0 == col1, only keep
    that indexing), plus an optional pool of short items handed out dynamically."""
    cases = [(np.array([0, 300, 300, 1000]), np.array([0, 5000, 5600, 9000]), 148),
             (np.arange(0, 1001, 10), np.arange(0, 16001, 160), 148),           # 100 classes of 10 queries
             (np.array([0, 7]), np.array([0, 50]), 148),
             (np.arange(0, 10001, 1000), np.arange(0, 60001, 6000), 148),       # C2 histogram
             (np.array([0, 5000, 5000, 5001]), np.array([0, 10, 4000, 4100]), 7)]
    for q_off, t_off, n_cta in cases:
        m, n = int(q_off[-1]), int(t_off[-1])
        classes = len(q_off) - 1
        q_class = np.repeat(np.arange(classes), np.diff(q_off))
        for mode, mixed, pool_frac in (("same", False, 0.0), ("other", False, 0.0), ("other", True, 0.0),
                                       ("same", False, 0.2), ("other", False, 0.2), ("other", True, 0.2)):
            ranges = [[(t_off[c], t_off[c + 1])] if mode == "same" else [(0, t_off[c]), (t_off[c + 1], t_off[-1])]
                      for c in range(classes)]
            tiles = E.query_tiles(q_off, ranges, t_off, 256, mixed)
            items, n_static = E.build_balanced_items(tiles, 256, n_cta, pool_frac=pool_frac, pool_tiles=4)
            assert 0 <= n_static <= items.shape[0] and (pool_frac > 0 or n_static == items.shape[0])
            pool = items[n_static:]
            assert np.all(pool[:, 3] > pool[:, 2]) and np.all(-(-(pool[:, 3] - pool[:, 2]) // 256) <= 4)
            live = items[items[:, 3] > items[:, 2]]
            total_tiles = int(np.sum(-(-(live[:, 3] - live[:, 2]) // 256)))
            cover = np.zeros((m, n), dtype=np.int32)
            for q0, rows, c0, c1, _, flag in live:
                assert 1 <= rows <= 256
                block = np.ones((rows, c1 - c0), dtype=np.int32)
                if flag & 1:
                    for r in range(rows):
                        c = q_class[q0 + r]
                        lo, hi = max(t_off[c], c0), min(t_off[c + 1], c1)
                        if hi > lo:
                            block[r, lo - c0:hi - c0] = 0
                else:
                    assert len(set(q_class[q0:q0 + rows])) == 1
                cover[q0:q0 + rows, c0:c1] += block
            want = np.zeros((m, n), dtype=np.int32)
            for c in range(classes):
                for lo, hi in ranges[c]:
                    want[q_off[c]:q_off[c + 1], lo:hi] = 1
            assert np.array_equal(cover, want), (mode, mixed, pool_frac)
            if items.shape[0] == 0:
                continue
            # the kernel's static schedule: grid = min(#items, #SMs), CTA b takes items b, b + grid, ...
            grid = min(items.shape[0], n_cta)
            load = np.zeros(grid, dtype=np.int64)
            for i, it in enumerate(items[:n_static]):
                load[i % grid] += -(-(it[3] - it[2]) // 256)
            static_tiles = int(load.sum())
            if total_tiles >= E.POOL_MIN_TILES * n_cta:
                assert load.max() <= np.ceil(static_tiles / grid) + 3, (load.max(), static_tiles / grid)
                assert load.min() >= np.floor(static_tiles / grid) - 3
                if pool_frac > 0:
                    assert 0.1 * total_tiles <= total_tiles - static_tiles <= 0.3 * total_tiles
    assert E.build_balanced_items([], 256, 148)[0].shape == (0, 6)


def test_shard_rows_partition_preserves_class_order():
    labels = np.random.default_rng(1).integers(0, 5, size=1003)
    parts = [E.shard_rows(labels, 5, r, 4) for r in range(4)]
    allrows = np.sort(np.concatenate(parts))
    assert np.array_equal(allrows, np.arange(1003))
    for p in parts:
        assert np.all(np.diff(p) > 0)
        counts = np.bincount(labels[p], minlength=5)
        assert np.all(np.abs(counts - np.bincount(labels, minlength=5) / 4) <= 1)


# ------------------------------------------------------------------------------------------
# world_size-2 gloo: the N_train-sharded protocol reproduces the single-shard oracle
# ------------------------------------------------------------------------------------------
def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        comm = E.TrainShardComm()
        xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(400, 60, 12, 3, seed=5)
        xtr[200:210] = xtr[0:10]                         # exact duplicates: tie-break on index
        ytr[200:210] = ytr[0:10]
        xte[:10] = xtr[0:10]
        pte[:10] = ytr[0:10]
        ytr[ytr == 2][:0]                                 # no-op
        keep = E.shard_rows(ytr, 3, rank, world)
        full = np_oracle.dsa_oracle(xtr, ytr, xte, pte)
        # per-shard stage 1 with the oracle (stands in for the CUDA search)
        da = np.full(60, np.nan, dtype=np.float32)
        gid = np.full(60, -1, dtype=np.int64)
        rows = np.zeros((60, 12), dtype=np.float32)
        for i in range(60):
            cand = keep[ytr[keep] == pte[i]]
            if cand.size:
                d = np.linalg.norm(xte[i][None, None, :] - xtr[cand][None], axis=2)[0]
                j = int(np.argmin(d))
                da[i], gid[i], rows[i] = d[j], cand[j], xtr[cand[j]]
        g_da, g_gid, g_rows = comm.reduce_winners(torch.from_numpy(da), torch.from_numpy(gid), torch.from_numpy(rows))
        assert np.array_equal(g_da.numpy(), full["dist_a"])
        assert np.array_equal(g_gid.numpy(), full["idx_a"])
        assert np.array_equal(g_rows.numpy(), xtr[full["idx_a"]])
        # float32 distances travel as ONE MIN all-reduce of packed (float bits << 32 | index) keys
        before = comm.collectives
        k_da, k_gid = comm.reduce_winner_index(torch.from_numpy(da), torch.from_numpy(gid))
        assert comm.collectives == before + 1
        assert np.array_equal(k_da.numpy(), full["dist_a"]) and np.array_equal(k_gid.numpy(), full["idx_a"])
        # ... and the winners come from the replicated training set by index: no row exchange at all
        before = comm.collectives
        r_da, r_gid, r_rows = comm.reduce_winners(torch.from_numpy(da), torch.from_numpy(gid), None, torch.from_numpy(xtr))
        assert comm.collectives == before + 1 and np.array_equal(r_rows.numpy(), xtr[full["idx_a"]])
        # float64: MIN of the distances, then MIN of the index among the holders of the minimum
        d_da, d_gid = comm.reduce_winner_index(torch.from_numpy(da.astype(np.float64)), torch.from_numpy(gid))
        assert np.array_equal(d_da.numpy(), full["dist_a"].astype(np.float64)) and np.array_equal(d_gid.numpy(), full["idx_a"])
        # a class nobody holds: NaN / -1 on every rank, both dtypes
        for dt in (torch.float32, torch.float64):
            e_d, e_g = comm.reduce_winner_index(torch.tensor([float("nan"), 2.0 + rank], dtype=dt),
                                                torch.tensor([-1, 7 + rank]))
            assert np.isnan(e_d[0].item()) and e_g[0].item() == -1 and e_d[1].item() == 2.0 and e_g[1].item() == 7
        # stage 2 on the shard: distance from the winning TRAIN rows to other-class rows
        db = np.full(60, np.nan, dtype=np.float32)
        for i in range(60):
            cand = keep[ytr[keep] != pte[i]]
            if cand.size:
                db[i] = np.linalg.norm(g_rows.numpy()[i][None, None, :] - xtr[cand][None], axis=2).min()
        g_db = comm.reduce_min_nan(torch.from_numpy(db))
        assert np.array_equal(g_db.numpy(), full["dist_b"])
        assert np.array_equal((g_da / g_db).numpy().astype(np.float64), full["dsa"])
        # LSE merge: per-shard (max, sum) -> global
        vals = np.random.default_rng(7).normal(size=(60, 400)) * 30 - 200
        mine = vals[:, rank::world]
        mx = mine.max(axis=1)
        sm = np.exp(mine - mx[:, None]).sum(axis=1)
        gm, gs = comm.reduce_lse(torch.from_numpy(mx), torch.from_numpy(sm))
        want = np.log(np.exp(vals - vals.max(axis=1, keepdims=True)).sum(axis=1)) + vals.max(axis=1)
        np.testing.assert_allclose(gm.numpy() + np.log(gs.numpy()), want, rtol=1e-12)
        # a class missing on one shard / everywhere
        nan_case = comm.reduce_min_nan(torch.tensor([float("nan"), 1.0 + rank]))
        assert np.isnan(nan_case[0].item()) and nan_case[1].item() == 1.0
        # a real +inf distance (squared differences that overflow) is a row, not "no row": it survives the exchange
        inf, nan = float("inf"), float("nan")
        for dt in (torch.float32, torch.float64):
            own = [inf, inf, nan, inf, nan] if rank == 0 else [nan, inf, nan, 5.0, -nan]
            g = comm.reduce_min_nan(torch.tensor(own, dtype=dt))
            assert g.dtype == dt and list(g[[0, 1, 3]].tolist()) == [inf, inf, 5.0] and np.isnan(g[[2, 4]].numpy()).all()
            i_d, i_g = comm.reduce_winner_index(torch.tensor([inf, inf, nan, inf], dtype=dt),
                                                torch.tensor([4 + rank, 9 - rank, -1, -1 if rank else 3]))
            assert i_d.dtype == dt and i_d[[0, 1, 3]].tolist() == [inf, inf, inf] and np.isnan(i_d[2].item())
            assert i_g.tolist() == [4, 8, -1, 3]
        # stage 1 -> stage 2 with every training row far out: the winners' traces are gathered, dist_b = inf
        big = np.full((4, 3), 3e19, dtype=np.float32)
        big[1] = 0.0
        w_da, w_gid, w_rows = comm.reduce_winners(torch.tensor([inf, 0.0] if rank == 0 else [inf, nan]),
                                                  torch.tensor([2 + rank, 1] if rank == 0 else [2 + rank, -1]),
                                                  None, torch.from_numpy(big))
        assert w_da.tolist() == [inf, 0.0] and w_gid.tolist() == [2, 1]
        assert np.array_equal(w_rows.numpy(), big[[2, 1]])
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_train_shard_protocol_gloo_world2():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(msg == "ok" for _, msg in results), results


def test_balanced_items_random_histograms_property():
    """Property check of the resident kernel's planner over random class histograms: whatever the
    shapes, every (query, train row) pair a stage needs is covered exactly once, items respect the
    tile height, pool items are short and real, and padding never carries work."""
    hypothesis = pytest.importorskip("hypothesis")
    from hypothesis import given, settings
    from hypothesis import strategies as st

    @settings(max_examples=60, deadline=None)
    @given(st.lists(st.integers(0, 700), min_size=1, max_size=6), st.lists(st.integers(0, 900), min_size=1, max_size=6),
           st.sampled_from([1, 7, 148]), st.sampled_from([64, 192, 256]), st.booleans(), st.sampled_from([0.0, 0.2, 0.5]))
    def check(q_counts, t_counts, n_cta, col_tile, mixed, pool_frac):
        classes = min(len(q_counts), len(t_counts))
        q_off = np.concatenate(([0], np.cumsum(q_counts[:classes])))
        t_off = np.concatenate(([0], np.cumsum(t_counts[:classes])))
        m, n = int(q_off[-1]), int(t_off[-1])
        q_class = np.repeat(np.arange(classes), np.diff(q_off))
        for mode in ("same", "other"):
            if mixed and mode == "same":
                continue
            ranges = [[(t_off[c], t_off[c + 1])] if mode == "same" else [(0, t_off[c]), (t_off[c + 1], t_off[-1])]
                      for c in range(classes)]
            tiles = E.query_tiles(q_off, ranges, t_off, 256, mixed)
            items, n_static = E.build_balanced_items(tiles, col_tile, n_cta, pool_frac=pool_frac, pool_tiles=3)
            assert items.dtype == np.int32 and items.shape[1] == 6 and 0 <= n_static <= items.shape[0]
            cover = np.zeros((m, n), dtype=np.int32)
            for q0, rows, c0, c1, _, flag in items:
                if c1 <= c0:
                    assert (q0, rows, c0, c1, flag) == (0, 0, 0, 0, 0)       # padding entry
                    continue
                assert 1 <= rows <= 256 and 0 <= c0 < c1 <= n and q0 + rows <= m
                block = np.ones((rows, c1 - c0), dtype=np.int32)
                if flag & 1:
                    for r in range(rows):
                        c = q_class[q0 + r]
                        lo, hi = max(t_off[c], c0), min(t_off[c + 1], c1)
                        if hi > lo:
                            block[r, lo - c0:hi - c0] = 0
                cover[q0:q0 + rows, c0:c1] += block
            want = np.zeros((m, n), dtype=np.int32)
            for c in range(classes):
                for lo, hi in ranges[c]:
                    want[q_off[c]:q_off[c + 1], lo:hi] = 1
            assert np.array_equal(cover, want)
            pool = items[n_static:]
            assert np.all(pool[:, 3] > pool[:, 2]) and np.all(-(-(pool[:, 3] - pool[:, 2]) // col_tile) <= 3)

    check()


def test_winner_keys_order_like_numpy_argmin():
    """Packed (float bits << 32 | index) keys: integer order == (distance, first occurrence)."""
    import torch

    rng = np.random.default_rng(11)
    d = np.abs(rng.normal(size=4096)).astype(np.float32)
    d[::7] = d[0]                                 # exact ties
    d[5] = 0.0
    d[9] = np.float32(1e-45)                      # subnormal
    d[100:4096:301] = np.inf                      # a real distance whose squares overflowed, tied among themselves
    gid = rng.permutation(4096).astype(np.int64)
    keys = E.pack_winner_keys(torch.from_numpy(d), torch.from_numpy(gid))
    assert (keys >= 0).all()
    order = np.lexsort((gid, d))
    assert np.array_equal(np.argsort(keys.numpy(), kind="stable"), order)
    back_d, back_g = E.unpack_winner_keys(keys)
    assert np.array_equal(back_d.numpy(), d) and np.array_equal(back_g.numpy(), gid)
    none = E.pack_winner_keys(torch.tensor([float("nan"), 1.0, -float("nan"), float("inf")]), torch.tensor([3, -1, 4, -1]))
    assert (none > keys.max()).all()
    nd, ng = E.unpack_winner_keys(none)
    assert np.isnan(nd.numpy()).all() and (ng.numpy() == -1).all()
    # the distance-only keys of the other exchanges: same order, +inf below "none", both dtypes
    for dt in (torch.float32, torch.float64):
        v = torch.tensor([0.0, 1e-300 if dt == torch.float64 else 1e-45, 2.0, float("inf"), float("nan"), -float("nan")],
                         dtype=dt)
        k = E.dist_keys(v)
        assert k.dtype == (torch.int32 if dt == torch.float32 else torch.int64)
        assert (k[:3] < k[3]).all() and (k[3] < k[4]).all() and k[4] == k[5]
        back = E.keys_dist(k)
        assert back.dtype == dt and back[:4].tolist() == v[:4].tolist() and torch.isnan(back[4:]).all()


def test_bench_clock_sampler_reports_rows_of_the_timed_region():
    """bench.py's nvidia-smi sampler: rows from before the timed region are ignored once rows inside exist, throttle
    reasons are collected, and a run whose sampler delivered nothing inside still reports the latest rows."""
    import time

    import bench

    s = bench.ClockSampler(0)
    s.proc = type("P", (), {"terminate": lambda self: None})()
    now = time.perf_counter()
    row = lambda sm, cap: ["0", str(sm), "1965", "500.0", "Not Active", "Not Active", "Not Active", cap]
    s.rows = [(now - 5.0, row(210, "Not Active")), (now - 4.9, row(1500, "Not Active"))]
    s.t_mark = now - 1.0
    s.rows += [(now - 0.5, row(1965, "Active")), (now - 0.4, row(1950, "Not Active")), (now - 0.3, row(1965, "Not Active"))]
    out = s.stop()
    assert out["samples_inside_timed_region"] == 3 and out["samples"] == 3
    assert out["sm_mhz"] == 1965.0 and out["sm_max_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"]
    s2 = bench.ClockSampler(0)
    s2.proc = type("P", (), {"terminate": lambda self: None})()
    s2.rows = [(now - 5.0, row(1800, "Not Active"))]
    s2.t_mark = now
    out2 = s2.stop()
    assert out2["samples_inside_timed_region"] == 0 and out2["samples"] == 1 and out2["sm_mhz"] == 1800.0
