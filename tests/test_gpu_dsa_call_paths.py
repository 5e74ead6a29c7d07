"""Every way DSA.__call__ produces a result runs the same launch sequence, `engine.dsa_scores`, and divides on the
device: the first (eager) call of a batch shape, the replayed CUDA-graph plan and a call with graphs switched off give
the same bytes — NaN bit patterns included — for the score, dist_a, dist_b and the winner index, and equal the
brute-force oracle."""
import numpy as np
import pytest

from oracle import c_oracle, np_oracle

pytestmark = pytest.mark.gpu


def _zero_over_zero(dt):
    """Training rows duplicated into another class: a test row equal to one has dist_a = dist_b = 0."""
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(3000, 300, 32, 3, seed=83, dtype=dt)
    xtr[10:20], ytr[10:20] = xtr[0:10], (ytr[0:10] + 1) % 3
    xte[:10], pte[:10] = xtr[0:10], ytr[0:10]
    xte[10:20], pte[10:20] = xtr[0:10], ytr[10:20]
    return xtr, ytr, xte, pte


def _heavy_ties():
    rng = np.random.default_rng(9)
    base = rng.integers(0, 2, size=(40, 16)).astype(np.float32)
    xtr = np.tile(base, (30, 1))                       # every row 30 times
    ytr = np.tile(np.arange(40) % 2, 30).astype(np.int64)
    xte = rng.integers(0, 2, size=(300, 16)).astype(np.float32)
    pte = rng.integers(0, 2, size=300).astype(np.int64)
    return xtr, ytr, xte, pte


def _case(name):
    """(xtr, ytr, xte, pte) of each case."""
    synth = lambda *a, dt=np.float32: np_oracle.synth_clusters(*a, dtype=dt)[:4]       # noqa: E731
    if name == "f32_resident":
        return synth(4000, 300, 64, 4, 71)
    if name == "f64_resident":
        return synth(4000, 300, 96, 5, 72, dt=np.float64)
    if name in ("f32_streaming", "f64_streaming"):
        return synth(3000, 400, 256, 4, 73, dt=np.float32 if name == "f32_streaming" else np.float64)
    if name in ("f32_distinct_winners", "table"):
        return synth(6000, 2000, 128, 4, 74)
    if name == "unscored_labels":
        xtr, ytr, xte, pte = synth(4000, 500, 64, 4, 75)
        pte[::7] = 4 + np.arange(pte[::7].size) % 3       # labels >= num_classes
        return xtr, ytr, xte, pte
    if name == "promoted":
        xtr, ytr, xte, pte = synth(3000, 260, 40, 4, 76)
        return xtr, ytr, xte.astype(np.float64) + 1e-9, pte
    if name == "cap1":
        return _heavy_ties()
    if name in ("zero_over_zero_f32", "zero_over_zero_f64"):
        return _zero_over_zero(np.float32 if name.endswith("f32") else np.float64)
    raise ValueError(name)


def _results(sa, got):
    return [got.copy(), sa.last_dist_a, sa.last_dist_b, sa.last_winner_index]


@pytest.mark.parametrize("name", ["f32_resident", "f64_resident", "f32_streaming", "f64_streaming",
                                  "f32_distinct_winners", "table", "unscored_labels", "promoted", "cap1",
                                  "zero_over_zero_f32", "zero_over_zero_f64"])
def test_eager_replayed_and_graphless_calls_give_the_same_bytes(name, monkeypatch):
    from simple_tip_b200 import engine as E
    from src.core.surprise import DSA

    calls = []
    dsa_scores = E.dsa_scores

    def spy(*args, **kwargs):
        calls.append(1)
        return dsa_scores(*args, **kwargs)

    monkeypatch.setattr(E, "dsa_scores", spy)
    xtr, ytr, xte, pte = _case(name)
    sa = DSA(xtr, ytr)
    if name == "table":
        sa.fit_other_class_table()
    if name == "cap1":
        sa._engine.cap = 1            # every query with more than one candidate chunk overflows its list
    if name == "f32_distinct_winners":
        _, q_off = E.class_layout(pte, int(sa.num_classes))
        assert sa._engine.distinct_ok(q_off, pte.shape[0])
    counts = []
    first = _results(sa, sa(xte, pte))
    counts.append(len(calls))
    sa(xte, pte)                      # the second sighting captures the plan
    counts.append(len(calls))
    sa._engine.stats.zero_()
    third = _results(sa, sa(xte, pte))
    counts.append(len(calls))
    overflow_rows = int(sa._engine.stats[0].item())
    sa.use_graphs = False
    graphless = _results(sa, sa(xte, pte))
    counts.append(len(calls))

    if name == "promoted":            # scored eagerly on two engines, never through a plan
        assert counts == [0, 0, 0, 0] and len(sa._engine._plans) == 0
        want = np_oracle.dsa_oracle(xtr, ytr, xte, pte)
        # stage 1 runs in float64 on the widened training traces; the NumPy oracle stores dist_a in the training dtype
        want["dist_a"] = c_oracle.dsa(xtr.astype(np.float64), ytr, xte, pte)["dist_a"]
    else:
        # the eager call and the plan's capture (a warm-up run and the captured run) go through dsa_scores; with
        # cap = 1 the replayed plan overflows, and the call is repeated eagerly through it
        assert counts == ([1, 4, 5, 6] if name == "cap1" else [1, 3, 3, 4]), counts
        assert len(sa._engine._plans) == 1
        assert (overflow_rows > 0) == (name == "cap1"), overflow_rows
        want = c_oracle.dsa(xtr, ytr, xte, pte)
    for a, b, c in zip(first, third, graphless):
        assert a.dtype == b.dtype == c.dtype
        assert a.tobytes() == b.tobytes() == c.tobytes()
    dsa, dist_a, dist_b, winner = first
    assert np.array_equal(winner, want["idx_a"])
    assert np.array_equal(dist_a, want["dist_a"], equal_nan=True)
    assert np.array_equal(dist_b, want["dist_b"], equal_nan=True)
    assert np.array_equal(dsa, want["dsa"], equal_nan=True)
    if name.startswith("zero_over_zero"):
        assert np.isnan(dsa[:20]).all() and (dist_a[:20] == 0).all() and (dist_b[:20] == 0).all()
    if name == "unscored_labels":
        assert np.isnan(dsa[::7]).all() and (winner[::7] == -1).all()
