"""The DSA filter (tip_nn_filter, pair_kernel<MODE_NN, ...> in csrc/pair_tc.cu) against a float64 model of its own
packed operands (oracle/filter_oracle.py), through the C ABI.  Per call the model checks the two properties DSA's
exactness rests on (DESIGN.md §4): every row's shared minimum is the minimum of its range's accumulators within the
accumulation slack, and every column inside the final window appears in some candidate mask; and that every list is
well formed (non-empty masks, bits inside the row's range, no column twice) and every admitted column sound.

Every kernel variant is reached through d alone: the resident kernel with the query tile's A operand from shared
memory (d <= 112), with K16 steps 1-7 from registers (k16 = 9: 113 <= d <= 128), and the streaming kernel (d > 128).
Each case runs DSA's three searches (same class; other classes with class-aligned query tiles; other classes with
tiles that mix classes and flagged items, whose exclusion cuts chunks mid-way) through the engine's planners (static
and pooled balanced lists at several CTA counts, or the streaming kernel's span-major lists) and through hand-built
lists within the header's contract: odd query-tile starts, spans that start and end mid-chunk, empty items,
consecutive items of one CTA that alternate query tiles (the resident reload and, at k16 = 9, the register reload),
one row's range split over several CTAs, rows no item covers.  Windows from measured rounding norms and from the
a-priori bound; running minima seeded as DSA's stage-2 hand-over does; cap 1 and 2 under planted many-way ties.

The data are clustered rows with planted structure: exact duplicates of a query's nearest row across chunk, tile and
item edges and in another class, rows on a ladder of distances up to the window's edge (completeness then requires
columns beyond the argmin), and in two cases a class whose rows approach the queries along the scan (event storms).
Every output buffer starts as 0xAB bytes and is followed by a guard region; the pool counters must be back at zero;
row_min_bits must be bit-identical across launches and schedules that scan the same pairs."""
import time

import numpy as np
import pytest

from oracle import filter_oracle as FO

pytestmark = pytest.mark.gpu

GUARD = 256
FILL = 0xAB
SAME, OTHER, MIXED = "same", "other", "mixed"


def _env():
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    return torch, _lib, _lib.load(), E


class Buf:
    """`nbytes` of device memory followed by a guard region; every byte 0xAB, or the payload zero-filled."""

    def __init__(self, nbytes, zero=False):
        torch = _env()[0]
        self.n = int(nbytes)
        self.t = torch.full((self.n + GUARD,), FILL, dtype=torch.uint8, device="cuda")
        if zero:
            self.t[:self.n].zero_()

    @property
    def ptr(self):
        return self.t.data_ptr()

    def get(self, dtype, shape=None):
        a = self.t[:self.n].cpu().numpy().view(dtype)
        return a if shape is None else a.reshape(shape)

    def put(self, a):
        torch = _env()[0]
        b = np.ascontiguousarray(a).view(np.uint8)
        assert b.size == self.n
        self.t[:self.n].copy_(torch.from_numpy(b.copy()))

    def guard_ok(self):
        return bool((self.t[self.n:] == FILL).all().item())


# ---- data ----------------------------------------------------------------------------------------------------------
def _data(rng, d, sizes, m, dtype, storm):
    """Train rows grouped by class (offsets class_off) and m class-sorted queries, with planted structure."""
    sizes = np.asarray(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n, C = int(off[-1]), len(sizes)
    centres = rng.normal(size=(C, d)) * 3.0
    cls = np.repeat(np.arange(C), sizes)
    t = centres[cls] + rng.normal(size=(n, d))
    if storm:
        # the biggest class's rows approach its centre along the scan: nearly every tile moves a query's minimum
        c = int(np.argmax(sizes))
        u = rng.normal(size=(sizes[c], d))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        t[off[c]:off[c + 1]] = centres[c] + u * np.linspace(20.0, 0.5, sizes[c])[:, None]
    pop = np.flatnonzero(sizes > 0)
    q_class = np.sort(rng.choice(pop, size=m))
    if storm:
        q_class[: m // 2] = int(np.argmax(sizes))
        q_class = np.sort(q_class)
    x = np.empty((m, d))
    delta = 0.05 * np.sqrt(d)
    for i, c in enumerate(q_class):
        if storm and c == int(np.argmax(sizes)):
            x[i] = centres[c] + rng.normal(size=d) * 0.01
        else:
            x[i] = t[rng.integers(off[c], off[c + 1])] + rng.normal(size=d) * delta / np.sqrt(d)
    # planted rows for a few queries: duplicates of the nearest row across chunk / tile / item edges and in another
    # class, and a ladder of distances d0 (1 + 2^-k) that reaches into the window's edge
    for i in rng.choice(m, size=min(m, 6), replace=False):
        c = int(q_class[i])
        lo, hi = int(off[c]), int(off[c + 1])
        j0 = lo + int(np.argmin(np.linalg.norm(t[lo:hi] - x[i], axis=1)))
        for step in (32, 96, 128, 129, 257):
            for p in (j0 + step, j0 - step):
                if lo <= p < hi:
                    t[p] = t[j0]
        others = [k for k in pop if k != c]
        if others:
            c2 = int(rng.choice(others))
            lo2, hi2 = int(off[c2]), int(off[c2 + 1])
            for p in {lo2, lo2 + 31, lo2 + 32, lo2 + 127, lo2 + 128, hi2 - 1}:
                if lo2 <= p < hi2:
                    t[p] = t[j0]
        d0 = max(float(np.linalg.norm(t[j0] - x[i])), 1e-3)
        for k in range(1, 14):
            u = rng.normal(size=d)
            y = x[i] + u / np.linalg.norm(u) * d0 * (1 + 2.0 ** -k)
            for a, b in ((lo, hi),) + (((lo2, hi2),) if others else ()):
                if b - a > 8:
                    p = int(rng.integers(a, b))
                    if not np.array_equal(t[p], t[j0]):
                        t[p] = y
    return t.astype(dtype), off, x.astype(dtype), q_class.astype(np.int32)


# ---- one filter call -----------------------------------------------------------------------------------------------
class Setup:
    """Engine (train operands), the queries' prepared state read back once, and the oracle's accumulators."""

    def __init__(self, t, off, x, q_class):
        torch, _lib, lib, E = _env()
        self.eng = E.NnEngine(torch.from_numpy(t).cuda(), off, torch.arange(t.shape[0], dtype=torch.int32).cuda(),
                              seeds=False)
        eng = self.eng
        self.lib, self.E, self.torch = lib, E, torch
        self.m, self.d, self.n = x.shape[0], eng.d, eng.n
        self.x = torch.from_numpy(x).cuda()
        self.q_class, self.off = q_class, off
        self.q_class_dev = torch.from_numpy(q_class).cuda()
        self.q_off = np.searchsorted(q_class, np.arange(len(off))).astype(np.int64)
        self.sms = eng.sms
        t_pack = eng.t_pack.view(torch.int16).cpu().numpy().view(np.uint16)
        # the window's t_rmax bounds every packed train row: |h(y)| = |packed[:d]| / 2 (scale -2 is exact)
        h = FO.bf16_bits(t_pack[:, :self.d]) / 2.0
        assert eng.rmax >= float(np.sqrt(np.max(np.sum(h * h, axis=1))))
        p = self.prep()
        self.q_pack = p["pack"].get(np.uint16, (self.m, eng.pitch))
        self.q_sq, self.q_err = p["sq"].get(np.float32), p["err"].get(np.float32)
        assert np.all(p["row_min"].get(np.uint32) == FO.INF_BITS) and np.all(p["cnt"].get(np.int32) == 0)
        self.a, self.slack = FO.accumulators(self.q_pack, t_pack, self.d)
        self.rmax, self.errmax = np.float32(eng.rmax), np.float32(eng.errmax)
        self.win = {True: FO.window(self.q_sq, self.q_err, self.rmax, self.errmax, self.d),
                    False: FO.window(self.q_sq, None, self.rmax, self.errmax, self.d)}

    def prep(self):
        m, eng = self.m, self.eng
        b = {"pack": Buf(m * eng.pitch * 2), "sq": Buf(4 * m), "err": Buf(4 * m), "row_min": Buf(4 * m),
             "cnt": Buf(4 * m)}
        rc = self.lib.tip_nn_query_prep(self.x.data_ptr(), eng.dtype, m, self.d, eng.center.data_ptr(), b["pack"].ptr,
                                        b["sq"].ptr, b["err"].ptr, b["row_min"].ptr, b["cnt"].ptr, None,
                                        self.torch.cuda.current_stream().cuda_stream)
        assert rc == 0, self.lib.tip_last_error()
        return b

    def run(self, items, n_static, flagged, measured=True, cap=None, seed_bits=None):
        """One tip_nn_filter call on freshly prepared query state; returns the checker's report and row_min_bits."""
        torch, lib, eng, m = self.torch, self.lib, self.eng, self.m
        cap = cap or eng.cap
        b = self.prep()
        if seed_bits is not None:
            b["row_min"].put(seed_bits.astype(np.uint32))
        idx = Buf(m * cap * 8)
        sched = Buf(8, zero=True)
        items = np.ascontiguousarray(items, dtype=np.int32).reshape(-1, 6)
        items_dev = torch.from_numpy(items).cuda()
        torch.cuda.synchronize()
        rc = lib.tip_nn_filter(b["pack"].ptr, b["sq"].ptr, m, eng.t_pack.data_ptr(), self.n, self.d, eng.pitch,
                               items_dev.data_ptr(), items.shape[0],
                               self.q_class_dev.data_ptr() if flagged else None,
                               eng.class_off_dev.data_ptr() if flagged else None, float(self.rmax),
                               b["err"].ptr if measured else None, float(self.errmax), b["row_min"].ptr, idx.ptr,
                               b["cnt"].ptr, cap, n_static, sched.ptr, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc == 0, lib.tip_last_error()
        for k, buf in list(b.items()) + [("cand_idx", idx), ("sched", sched)]:
            assert buf.guard_ok(), f"write past the end of {k}"
        assert np.all(sched.get(np.int32) == 0), "the pool counters are not back at zero"
        row_min, cnt = b["row_min"].get(np.uint32), b["cnt"].get(np.int32)
        cand = idx.get(np.int32, (m, cap, 2))
        inr, owner, times = FO.row_ranges(m, self.n, items, self.q_class if flagged else None,
                                          self.off if flagged else None)
        assert times.max(initial=0) <= 1, "the test's work list scans a pair twice"
        rep = FO.check(self.a, self.slack, self.win[measured], inr, owner, row_min, cand, cnt, cap,
                       seed_bits=seed_bits)
        # entries past min(cnt, cap) are never written
        for i in range(m):
            k = min(max(int(cnt[i]), 0), cap)
            assert np.all(cand[i, k:].view(np.uint32) == 0xABABABAB), f"row {i}: an entry past the count was written"
        return rep, row_min, cnt, cand, inr

    # ---- work lists ----
    def ranges(self, mode):
        off = self.off
        C = len(off) - 1
        if mode == SAME:
            return [[(off[c], off[c + 1])] for c in range(C)]
        return [[(0, off[c]), (off[c + 1], off[-1])] for c in range(C)]

    def planner_lists(self, mode):
        """(name, items, n_static) of the engine's planners for this kernel variant."""
        E = self.E
        ranges, mixed = self.ranges(mode), mode == MIXED
        if self.eng.resident:
            tiles = E.query_tiles(self.q_off, ranges, self.off, self.eng.row_tile, mixed)
            out = []
            for name, n_cta, frac in (("static", self.sms, 0.0), ("static5", 5, 0.0), ("pool1", 1, 0.3),
                                      ("pool3", 3, 0.2)):
                items, n_static = E.build_balanced_items(tiles, self.eng.col_tile, n_cta, pool_frac=frac, pool_tiles=4)
                out.append((name, items, n_static))
            # the planner pools only long lists: the static list again, its back half drawn through the counter
            items = out[0][1]
            out.append(("pool-half", items, items.shape[0] // 2))
            return out
        out = []
        for st in (1, 3):
            span_of = (lambda pairs, st=st: st)
            if mixed:
                items = E.build_other_class_items(self.q_off, self.off, self.eng.row_tile, self.eng.col_tile, span_of)
            else:
                items, _ = E.build_items(self.q_off, ranges, st, self.eng.row_tile, self.eng.col_tile)
            items = E.span_major(items)
            out.append((f"span{st}", items, items.shape[0]))
        return out

    def hand_list(self, mode, rng):
        """Query tiles of 70 rows (odd starts, partial tiles) x spans cut at random points (mid-chunk, some empty),
        ordered so that each CTA runs three consecutive entries that alternate query tiles.  The first tile is left
        out: its rows keep the prepared state."""
        E = self.E
        tiles = E.query_tiles(self.q_off, self.ranges(mode), self.off, 70, mode == MIXED)[1:]
        per_tile = []
        for r0, nr, rs, flag in tiles:
            spans = []
            for lo, hi in rs:
                cuts = np.unique(np.concatenate([[lo, hi], rng.integers(lo, hi + 1, size=max(1, (hi - lo) // 60))]))
                spans += [(int(a), int(b)) for a, b in zip(cuts[:-1], cuts[1:])]
                spans.append((int(hi), int(hi)))                   # col0 == col1
            per_tile.append([(r0, nr, a, b, 0, flag) for a, b in spans])
        seq = []
        for k in range(max((len(p) for p in per_tile), default=0)):
            seq += [p[k] for p in per_tile if len(p) > k]
        if not seq:
            return None
        R = max(3, -(-len(seq) // self.sms))
        seq += [(0, 0, 0, 0, 0, 0)] * (self.sms * R - len(seq))
        items = np.zeros((self.sms * R, 6), dtype=np.int32)
        for b in range(self.sms):
            for k in range(R):
                items[k * self.sms + b] = seq[b * R + k]
        return items


def _admitted(cand, cnt, cap, i):
    cols = set()
    for col, mask in cand[i, :min(int(cnt[i]), cap)]:
        mk = int(mask) & 0xFFFFFFFF
        cols |= {int(col) + b for b in range(32) if (mk >> b) & 1}
    return cols


# (d, dtype, class sizes, m, event storm): each width of the three kernel variants once
CASES = [
    (1, np.float32, [33, 0, 129, 31, 2], 63, False),
    (16, np.float64, [1, 127, 128, 300], 129, False),
    (17, np.float32, [1000, 33, 0, 200], 193, False),
    (48, np.float64, [129, 32, 500], 64, False),
    (97, np.float32, [31, 2, 1000, 1], 450, True),
    (112, np.float64, [300, 300], 1, False),
    (113, np.float32, [129, 1000, 33], 191, False),
    (120, np.float64, [32, 127, 0, 600], 65, False),
    (128, np.float32, [1000, 1000, 31], 450, True),
    (129, np.float64, [200, 33, 129], 128, False),
    (200, np.float32, [1000, 2, 127], 192, False),
    (1600, np.float32, [300, 129, 31], 129, False),
]
KIND = {d: (1 if d <= 128 else 0, -(-d // 16) + 1) for d in (1, 16, 17, 48, 97, 112, 113, 120, 128, 129, 200, 1600)}


def test_variant_boundaries():
    """The widths below reach the variants they are meant for: a change of the boundaries shows up here."""
    lib = _env()[2]
    for d, (kind, k16) in KIND.items():
        assert lib.tip_nn_filter_kind(d) == kind, d
        assert FO.k16_of(d) == k16
        assert (k16 == 9) == (113 <= d <= 128)


@pytest.mark.parametrize("d,dtype,sizes,m,storm", CASES,
                         ids=[f"d{c[0]}-{np.dtype(c[1]).name}-m{c[3]}{'-storm' if c[4] else ''}" for c in CASES])
def test_filter_against_float64_model(d, dtype, sizes, m, storm):
    t0 = time.perf_counter()
    rng = np.random.default_rng(1000 + d)
    s = Setup(*_data(rng, d, sizes, m, dtype, storm))
    worst, launches, required, outside, pooled = 0.0, 0, {}, 0, 0

    def run(tag, *args, **kw):
        nonlocal worst, launches, outside
        rep, row_min, cnt, cand, inr = s.run(*args, **kw)
        assert not rep.findings, f"{tag}:\n" + rep.summary()
        worst = max(worst, rep.rowmin_frac)
        launches += 1
        outside += rep.outside
        return rep, row_min, cnt, cand, inr

    ref = {}                  # row_min_bits by pair set: SAME, or the other-class range (OTHER and MIXED share it)
    for mode in (SAME, OTHER, MIXED):
        key = SAME if mode == SAME else OTHER
        flagged = mode == MIXED
        lists = s.planner_lists(mode)
        hand = s.hand_list(mode, rng)
        if hand is not None:
            lists.append(("hand", hand, hand.shape[0]))
            if s.eng.resident:
                lists.append(("hand-pool", hand, 0))
        required.setdefault(mode, 0)
        for li, (name, items, n_static) in enumerate(lists):
            if items.shape[0] == 0:
                continue
            pooled += name.startswith("pool") and n_static < items.shape[0]
            fl = flagged and bool((items[:, 5] & 1).any())
            runs = [(True, None)] + ([(True, None), (False, None)] if li == 0 else [])
            for measured, _ in runs:
                rep, row_min, cnt, cand, inr = run(f"{mode}/{name}/{'measured' if measured else 'a-priori'}",
                                                   items, n_static, fl, measured)
                required[mode] += rep.required_extra
                covered = inr.any(axis=1)
                if key in ref:
                    r0, c0 = ref[key]
                    both = covered & c0
                    assert np.array_equal(row_min[both], r0[both]), f"{mode}/{name}: row_min_bits differ by schedule"
                    # rows no item covers keep tip_nn_query_prep's state
                assert np.all(row_min[~covered] == FO.INF_BITS) and np.all(cnt[~covered] == 0)
                if key not in ref or covered.sum() > ref[key][1].sum():
                    ref[key] = (row_min.copy(), covered)
        assert required[mode] > 0, f"{mode}: nothing beyond the argmin was required"
    assert pooled > 0 or not s.eng.resident, "no list had a pool"

    # seeds: row_min preset as DSA's stage-2 hand-over does it, from the NumPy distance to one in-range row (the
    # argmin on even rows, any row on odd ones); with the window argument the argmin must be admitted
    name, items, n_static = s.planner_lists(OTHER)[0]
    if items.shape[0]:
        inr = FO.row_ranges(m, s.n, items)[0]
        xq, tt = s.x.cpu().numpy(), s.eng.t.cpu().numpy()
        gamma = np.float32(np.float32(16 * FO.k16_of(d) + 16) * np.float32(1.1920929e-7))
        seed = np.full(m, FO.INF_BITS, dtype=np.uint32)
        must = {}
        for i in np.flatnonzero(inr.any(axis=1)):
            cols = np.flatnonzero(inr[i])
            dist = np.linalg.norm(xq[i][None, None, :] - tt[cols][None], axis=2)[0]
            j = int(cols[np.argmin(dist)]) if i % 2 == 0 else int(rng.choice(cols))
            if i % 2 == 0:
                must[i] = j
            ub = np.float32(np.linalg.norm((xq[i] - tt[j])[None, None, :], axis=2)[0, 0])
            r = np.float32(np.sqrt(s.q_sq[i], dtype=np.float32) + s.rmax)
            e = np.float32(np.float32(s.q_err[i] + s.errmax + np.float32(1.2e-7) * r) * np.float32(1.00001))
            g = np.float32(gamma * r * r)
            dd = np.float32(np.float32(ub * np.float32(1.000004)) + e)
            seed[i] = np.float32(np.float32(dd * dd + g) * np.float32(1.000002)).view(np.uint32)
        rep, row_min, cnt, cand, _ = run("seeded", items, n_static, False, True, seed_bits=seed)
        for i, j in must.items():
            if cnt[i] <= s.eng.cap:
                assert j in _admitted(cand, cnt, s.eng.cap, i), f"seeded row {i}: its argmin {j} is not admitted"

    # overflow: cap 1 and 2 under the planted ties; the first cap entries stay well formed
    name, items, n_static = s.planner_lists(SAME)[0]
    overflowed = 0
    if items.shape[0]:
        for cap in (1, 2):
            rep = run(f"cap{cap}", items, n_static, False, True, cap=cap)[0]
            overflowed += rep.overflowed
        assert overflowed > 0 or m == 1, "no list overflowed"
    assert outside > 0, "no admitted chunk held a column outside its window"
    print(f"filter d={d} {np.dtype(dtype).name} m={m}: row_min worst error = {worst:.3g} of the bound; required beyond "
          f"the argmin {required}; outside-window columns of admitted chunks {outside}; overflowed rows {overflowed}; "
          f"{pooled} pooled lists; {launches} launches, {time.perf_counter() - t0:.1f} s")
