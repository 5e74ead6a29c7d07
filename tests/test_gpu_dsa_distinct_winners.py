"""DSA's stage 2 once per distinct stage-1 winner (tip_dsa_distinct_winners + tip_nn_filter_live).

Stage 2 searches from the winning train row, so inputs that share a winner share a search.  The scores must stay
NumPy's bits: every case is checked against the brute-force C oracle through the public DSA class (eager call,
graph capture, replays), and the compaction itself against a host restatement of its slots."""
import numpy as np
import pytest

from oracle import c_oracle, np_oracle

pytestmark = pytest.mark.gpu


def _copies(rng, xtr, ytr, cls, distinct, count, noise=1e-3):
    """`count` inputs of class `cls`, each a noisy copy of one of `distinct` train rows of that class (every one used)."""
    rows = rng.choice(np.flatnonzero(ytr == cls), size=distinct, replace=False)
    pick = np.concatenate([rows, rng.choice(rows, size=count - distinct)]) if count > distinct else rows
    x = xtr[pick] + (noise * rng.normal(size=(count, xtr.shape[1]))).astype(xtr.dtype)
    return x.astype(xtr.dtype), np.full(count, cls, dtype=np.int64)


def _dataset(kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "collapse":       # class 0: one winner; class 1: five; class 2: every winner distinct
        xtr, ytr, _, _, _ = np_oracle.synth_clusters(3000, 10, 64, 3, seed=seed)
        parts = [_copies(rng, xtr, ytr, 0, 1, 500), _copies(rng, xtr, ytr, 1, 5, 500),
                 _copies(rng, xtr, ytr, 2, 500, 500)]
    elif kind == "multiples":    # k_c = 192, 64, 384: whole 192-row tiles, whole 64-row warpgroup slices
        xtr, ytr, _, _, _ = np_oracle.synth_clusters(6000, 10, 128, 3, seed=seed)
        parts = [_copies(rng, xtr, ytr, 0, 192, 576), _copies(rng, xtr, ytr, 1, 64, 448),
                 _copies(rng, xtr, ytr, 2, 384, 384)]
    elif kind == "empty_class":  # class 2 of 4 has no inputs
        xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(8000, 2400, 128, 4, seed=seed)
        keep = pte != 2
        return xtr, ytr, xte[keep], pte[keep]
    elif kind == "synth":        # C2-like clusters: mostly distinct winners, some shared
        xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(6000, 2000, 128, 4, seed=seed)
        return xtr, ytr, xte, pte
    else:
        raise ValueError(kind)
    xte = np.concatenate([p[0] for p in parts])
    pte = np.concatenate([p[1] for p in parts])
    perm = rng.permutation(xte.shape[0])     # the caller's order is not class-sorted
    return xtr, ytr, np.ascontiguousarray(xte[perm]), pte[perm]


def _check(sa, xte, pte, want):
    got = sa(xte, pte)
    assert np.array_equal(sa.last_winner_index, want["idx_a"])
    assert np.array_equal(sa.last_dist_a, want["dist_a"], equal_nan=True)
    assert np.array_equal(sa.last_dist_b, want["dist_b"], equal_nan=True)
    assert np.array_equal(got, want["dsa"], equal_nan=True)


def _distinct_path(sa, pte):
    from simple_tip_b200 import engine as E

    _, q_off = E.class_layout(pte, int(sa.num_classes))
    return sa._engine.distinct_ok(q_off, pte.shape[0])


@pytest.mark.parametrize("kind", ["collapse", "multiples", "empty_class", "synth"])
def test_dsa_distinct_winners_vs_c_oracle(kind):
    from src.core.surprise import DSA

    xtr, ytr, xte, pte = _dataset(kind)
    want = c_oracle.dsa(xtr, ytr, xte, pte)
    sa = DSA(xtr, ytr)
    assert _distinct_path(sa, pte)
    for _ in range(3):           # eager, captured, replayed
        _check(sa, xte, pte, want)
    assert int(sa._engine.stats[0].item()) == 0, "rows fell back to the exhaustive scan"


def test_dsa_plan_replay_across_winner_counts():
    """One captured plan (same class histogram), inputs whose distinct-winner counts differ from call to call."""
    from src.core.surprise import DSA

    xtr, ytr, xa, pte = _dataset("multiples", seed=3)
    rng = np.random.default_rng(5)
    xb = xa.copy()
    for c in range(3):              # the same histogram, every class collapsed onto two rows
        sel = np.flatnonzero(pte == c)
        xb[sel] = _copies(rng, xtr, ytr, c, 2, sel.size)[0]
    xc = xtr[rng.choice(np.flatnonzero(ytr == 0), size=1)].repeat(pte.size, 0)   # every input near one point
    xc = xc + (0.5 * rng.normal(size=xc.shape)).astype(xc.dtype)
    sa = DSA(xtr, ytr)
    assert _distinct_path(sa, pte)
    wants = {k: c_oracle.dsa(xtr, ytr, x, pte) for k, x in (("a", xa), ("b", xb), ("c", xc))}
    for k in ("a", "a", "b", "c", "a", "b"):
        _check(sa, {"a": xa, "b": xb, "c": xc}[k], pte, wants[k])


@pytest.mark.parametrize("kind", ["collapse", "multiples", "empty_class"])
def test_distinct_winner_slots_vs_host(kind):
    """The compaction itself: slots in training-row order per class, k_c exact, every input's slot, the live bound,
    the winners' rows and their packed stage-2 query state."""
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    xtr, ytr, xte, pte = _dataset(kind, seed=1)
    classes = int(max(ytr.max(), pte.max())) + 1
    eng = E.NnEngine.from_host(xtr, ytr, classes)
    order, q_off = E.class_layout(pte, classes)
    m = pte.shape[0]
    assert eng.distinct_ok(q_off, m)
    x = E.to_device(xte[order], eng.dev)
    q_class = torch.from_numpy(pte[order].astype(np.int32)).to(eng.dev)
    _, pos, _, _ = eng.search(x, q_class, q_off, _lib.RANGE_SAME_CLASS)
    rows, state, slot_class, live_end, k, slot = eng.distinct_winners(pos, q_off)
    torch.cuda.synchronize()
    pos_h = pos.cpu().numpy()
    t_h = eng.t.cpu().numpy()
    k_h, slot_h, cls_h, end_h = (a.cpu().numpy() for a in (k, slot, slot_class, live_end))
    cnt_h = state[4].cpu().numpy()
    live = []
    for c in range(classes):
        q0, q1 = int(q_off[c]), int(q_off[c + 1])
        if q0 == q1:
            continue
        winners = np.unique(pos_h[q0:q1])          # ascending train position = training-row order inside the class
        assert winners.min() >= eng.class_off[c] and winners.max() < eng.class_off[c + 1]
        assert k_h[c] == winners.size
        np.testing.assert_array_equal(slot_h[q0:q1], q0 + np.searchsorted(winners, pos_h[q0:q1]))
        np.testing.assert_array_equal(end_h[q0:q1], q0 + winners.size)
        np.testing.assert_array_equal(cls_h[q0:q1], np.where(np.arange(q1 - q0) < winners.size, c, -1))
        np.testing.assert_array_equal(cnt_h[q0 + winners.size:q1], 0)
        np.testing.assert_array_equal(rows[q0:q0 + winners.size].cpu().numpy(), t_h[winners])
        live.extend(range(q0, q0 + winners.size))
    # the packed state of the live slots is tip_nn_query_prep's for the same rows (the seeds aside)
    live = torch.tensor(live, dtype=torch.int64, device=eng.dev)
    want = eng.query_state(live.numel())
    lr = rows.index_select(0, live).contiguous()
    _lib.check(eng.lib.tip_nn_query_prep(E._p(lr), E.tip_dtype(lr.dtype), lr.shape[0], eng.d, E._p(eng.center),
                                         E._p(want[0]), E._p(want[1]), E._p(want[2]), E._p(want[3]), E._p(want[4]),
                                         None, E._stream()), "tip_nn_query_prep")
    for got_t, want_t in zip(state[:3], want[:3]):
        assert torch.equal(got_t.index_select(0, live).view(torch.int16 if got_t.dtype == torch.bfloat16 else torch.int32),
                           want_t.view(torch.int16 if want_t.dtype == torch.bfloat16 else torch.int32))
