"""Pins oracle/rerank_oracle.py, the reference of the exact re-rank's C contract (csrc/rerank.cu), three ways:
against np_oracle.dsa_oracle and the C oracle when every candidate list names the whole range, against a
brute-force restatement of the list rules, and its pairwise-sum model against np.linalg.norm at every width the GPU
tests run.  Each comparison is also run with a defect injected into the oracle (ties to the highest index, the own
class admitted in OTHER mode, NumPy's split point not rounded to a multiple of 8) and must then fail."""
import numpy as np
import pytest

from oracle import c_oracle, np_oracle
from oracle import rerank_oracle as RO

f32, f64 = np.float32, np.float64


def _dsa_case(dt, seed=3):
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(300, 40, 9, 4, seed=seed)
    xtr, xte = xtr.astype(dt), xte.astype(dt)
    xtr[150:160] = xtr[0:10]                      # exact duplicates: ties broken by the original index
    ytr[150:160] = ytr[0:10]
    xte[:6] = xtr[150:156]
    pte[:6] = ytr[150:156]
    order = np.argsort(ytr, kind="stable")        # class-grouped, ascending original index inside a class
    class_off = np.concatenate(([0], np.cumsum(np.bincount(ytr, minlength=4))))
    return xtr, ytr, xte, pte, xtr[order], order.astype(np.int32), class_off


def _whole_range_lists(m, n):
    chunks = (n + 31) // 32
    idx = np.zeros((m, chunks, 2), dtype=np.int32)
    idx[:, :, 0] = np.arange(chunks) * 32
    idx[:, :, 1] = -1                              # all 32 bits
    return idx, np.full(m, chunks, dtype=np.int32), chunks


def _two_stages(dt, lists):
    xtr, ytr, xte, pte, t, gid, class_off = _dsa_case(dt)
    m, n = xte.shape[0], t.shape[0]
    kw = {}
    if lists:
        idx, cnt, cap = _whole_range_lists(m, n)
        kw = dict(cand_idx=idx, cand_cnt=cnt, cap=cap)
    a = RO.rerank(xte, t, class_off, pte, RO.SAME_CLASS, t_gid=gid, **kw)
    b = RO.rerank(a["out_rows"], t, class_off, pte, RO.OTHER_CLASSES, t_gid=gid, **kw)
    return (xtr, ytr, xte, pte), a, b


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("lists", [False, True])
def test_rerank_oracle_is_dsa_when_lists_name_the_whole_range(dt, lists):
    (xtr, ytr, xte, pte), a, b = _two_stages(dt, lists)
    for want in (np_oracle.dsa_oracle(xtr, ytr, xte, pte), c_oracle.dsa(xtr, ytr, xte, pte)):
        assert np.array_equal(a["out_dist"], want["dist_a"])
        assert np.array_equal(a["out_gid"], want["idx_a"])
        assert np.array_equal(b["out_dist"], want["dist_b"])
    assert np.array_equal(a["out_rows"], xtr[a["out_gid"]])
    assert a["scanned"] == (0 if lists else xte.shape[0])


def test_rerank_oracle_rejects_ties_to_the_highest_index(monkeypatch):
    monkeypatch.setattr(RO, "winner", lambda dist, gid: int(np.lexsort((-gid, dist))[0]))
    (xtr, ytr, xte, pte), a, _ = _two_stages(f32, True)
    assert not np.array_equal(a["out_gid"], np_oracle.dsa_oracle(xtr, ytr, xte, pte)["idx_a"])


def test_rerank_oracle_rejects_own_class_in_other_mode(monkeypatch):
    same = RO.in_range
    monkeypatch.setattr(RO, "in_range", lambda j, off, c, mode: same(j, off, c, mode) if mode == RO.SAME_CLASS
                        else j < int(off[-1]))
    (xtr, ytr, xte, pte), _, b = _two_stages(f64, False)
    assert not np.array_equal(b["out_dist"], np_oracle.dsa_oracle(xtr, ytr, xte, pte)["dist_b"])


# ---- the list rules, against a brute force ------------------------------------------------------------------
def _bruteforce(q, t, class_off, q_class, mode, cand_idx, cand_cnt, cap, t_gid):
    """One row at a time: a row is a candidate if some entry's mask names it (or the query has no usable list and
    the row is in range); distances from the scalar pairwise-sum model; the first (distance, gid) minimum wins."""
    n = t.shape[0]
    gids = np.arange(n) if t_gid is None else t_gid
    res = []
    for r in range(q.shape[0]):
        c = int(q_class[r])
        if not 0 <= c < len(class_off) - 1:
            res.append((None, -1))
            continue
        lo, hi, cn = class_off[c], class_off[c + 1], class_off[-1]
        ok = [(lo <= j < hi) if mode == RO.SAME_CLASS else (j < cn and not lo <= j < hi) for j in range(n)]
        cnt = int(cand_cnt[r])
        if 1 <= cnt <= cap:
            named = [False] * n
            for start, mask in cand_idx[r, :cnt]:
                for bit in range(32):
                    if (int(mask) >> bit) & 1 and 0 <= int(start) + bit < n:
                        named[int(start) + bit] = True
            ok = [o and nm for o, nm in zip(ok, named)]
        best = None
        for j in range(n):
            if ok[j]:
                diff = q[r] - t[j]
                dj = np.sqrt(np_oracle.pairwise_sum_model(diff * diff))
                if best is None or dj < best[0] or (dj == best[0] and gids[j] < gids[best[1]]):
                    best = (dj, j)
        res.append((None, -1) if best is None else best)
    return res


def _list_case(dt, d, seed):
    rng = np.random.default_rng(seed)
    n, m, cap = 70, 40, 3
    class_off = np.array([0, 0, 25, 26, 70])            # an empty class and a one-row class
    t = (rng.normal(size=(n, d)) * 3).astype(dt)
    t[40:44] = t[30]                                    # ties, resolved by a gid that reverses position order
    q = (rng.normal(size=(m, d)) * 3).astype(dt)
    q[:4] = t[30]
    q_class = rng.integers(-1, 5, size=m).astype(np.int32)        # -1 and 4 are invalid
    cnt = rng.integers(0, cap + 2, size=m).astype(np.int32)       # 0 and cap + 1: scanned
    idx = np.zeros((m, cap, 2), dtype=np.int32)
    idx[:, :, 0] = rng.integers(-40, n + 10, size=(m, cap))       # negative starts, bits past n
    idx[:, :, 1] = rng.integers(0, 1 << 32, size=(m, cap), dtype=np.int64).astype(np.uint32).view(np.int32)
    idx[::5, 0, 1] = 0                                            # empty masks
    idx[1::7, 1] = idx[1::7, 0]                                   # duplicate entries
    gid = np.arange(n)[::-1].astype(np.int32)
    return q, t, class_off, q_class, idx, cnt, cap, gid


@pytest.mark.parametrize("dt", [f32, f64])
@pytest.mark.parametrize("mode", [RO.SAME_CLASS, RO.OTHER_CLASSES])
def test_rerank_oracle_list_rules_match_bruteforce(dt, mode):
    for d, seed in ((5, 0), (37, 1)):
        q, t, class_off, q_class, idx, cnt, cap, gid = _list_case(dt, d, seed)
        got = RO.rerank(q, t, class_off, q_class, mode, idx, cnt, cap, t_gid=gid)
        want = _bruteforce(q, t, class_off, q_class, mode, idx, cnt, cap, gid)
        for r, (wd, wj) in enumerate(want):
            assert got["out_pos"][r] == wj, (d, r)
            if wj < 0:
                assert np.isnan(got["out_dist"][r]) and got["out_gid"][r] == -1 and not got["out_rows"][r].any()
            else:
                assert got["out_dist"][r] == wd and got["out_gid"][r] == gid[wj]
                assert np.array_equal(got["out_rows"][r], t[wj])
        valid = (q_class >= 0) & (q_class < 4)
        assert got["scanned"] == int((valid & ((cnt < 1) | (cnt > cap))).sum())
        assert (got["out_pos"] >= 0).any() and (got["out_pos"] < 0).any()


# ---- the pairwise-sum model against np.linalg.norm -----------------------------------------------------------------
def _pair(dt, d, seed):
    rng = np.random.default_rng(seed)
    x = (rng.normal(size=d) * 2 + 1).astype(dt)
    y = (rng.normal(size=d) * 2).astype(dt)
    return x, y


@pytest.mark.parametrize("dt", [f32, f64])
def test_norm_model_matches_numpy_at_every_kernel_width(dt):
    for d in RO.KERNEL_WIDTHS:
        x, y = _pair(dt, d, d)
        got, want = RO.norm_model(x, y), RO.norms(x, y[None])[0]
        assert got.dtype == want.dtype == dt and got == want, d
    for d in (7, 8, 9, 127, 128, 129, 300, 4100):
        x, y = _pair(dt, d, 1000 + d)
        diff = x - y
        assert RO.pairwise_sum(diff * diff) == np_oracle.pairwise_sum_model(diff * diff) == np.add.reduce(diff * diff)


def test_norm_model_rejects_an_unaligned_split(monkeypatch):
    monkeypatch.setattr(RO, "_split", lambda n: n // 2)
    bad = 0
    for d in (137, 143, 257, 263, 513, 1000, 1025, 2049, 4097, 8193):
        for seed in range(4):
            x, y = _pair(f32, d, seed)
            bad += RO.norm_model(x, y) != RO.norms(x, y[None])[0]
    assert bad > 0


def test_pack_query_model():
    rng = np.random.default_rng(4)
    x = rng.normal(size=(3, 21)).astype(f64)
    c = rng.normal(size=21).astype(f32)
    bits = RO.pack_query(x, c)
    assert bits.shape == (3, RO.pair_pitch(21)) == (3, 64)
    v = RO.bf16_values(bits)
    assert np.array_equal(v[:, 32:35], np.ones((3, 3))) and not v[:, 35:].any() and not v[:, 21:32].any()
    exact = (x - c.astype(f64)).astype(f32).astype(f64)
    assert np.all(np.abs(v[:, :21] - exact) <= np.abs(exact) * 2.0 ** -8)


def test_pack_out_model_divides_like_numpy():
    da = np.array([0, 1, np.inf, 2, 3, 9, 9], dtype=f32)
    db = np.array([0, 0, np.inf, np.inf, 2, 1, 1], dtype=f32)
    out = np.full((4, 6), -7.0)
    RO.pack_out(da, db, np.arange(7, dtype=np.int32), np.array([5, 1, 0, 3, 2, 6, -1]), 6, out)
    assert np.isnan(out[3, 5]) and out[3, 1] == np.inf and np.isnan(out[3, 0]) and out[3, 3] == 0.0
    assert out[3, 2] == 1.5 and np.all(out[:, 4] == -7.0)
    assert list(out[:3, 5]) == [0.0, 0.0, 0.0] and list(out[:3, 2]) == [3.0, 2.0, 4.0]
