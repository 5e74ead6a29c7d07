"""tip_keras_adam against a NumPy float32 restatement of its documented operation order, bit for bit, eagerly and
replayed from a captured graph; tip_softmax_xent against a float64 NumPy reference."""
import numpy as np
import pytest

from oracle.train_oracle import adam_restatement

pytestmark = pytest.mark.gpu

SIZES = (1, 3, 5, 1023, 4097, 1_600_000)
STEPS = 20
F = np.float32


def _tables(torch, E, rng):
    """Every tensor a slice of one buffer per role, at starts that give each tensor's four arrays equal or unequal
    alignments (the vector and the scalar route)."""
    dev = torch.device("cuda")
    total = sum(SIZES) + 8 * len(SIZES)
    bufs = {k: torch.zeros(total, dtype=torch.float32, device=dev) for k in ("p", "g", "m", "v")}
    views = {k: [] for k in bufs}
    pos = 0
    for i, n in enumerate(SIZES):
        for k in bufs:
            shift = (i + (1 if (k == "v" and i % 2) else 0)) % 4      # odd tensors: v misaligned against the rest
            views[k].append(bufs[k][pos + shift:pos + shift + n])
        pos += n + 8
    p0 = [rng.normal(size=n).astype(np.float32) for n in SIZES]
    for view, a in zip(views["p"], p0):
        view.copy_(torch.from_numpy(a))
    grads = [[rng.normal(size=n).astype(np.float32) * F(10.0 ** rng.integers(-3, 2)) for n in SIZES]
             for _ in range(STEPS)]
    table = E.adam_table(views["p"], views["g"], views["m"], views["v"])
    return views, table, p0, grads


def _check(views, p0, grads):
    for i in range(len(SIZES)):
        p, m, v = adam_restatement(p0[i], [g[i] for g in grads])
        assert np.array_equal(views["p"][i].cpu().numpy(), p), f"param of tensor {i} ({SIZES[i]} elements)"
        assert np.array_equal(views["m"][i].cpu().numpy(), m), f"m of tensor {i}"
        assert np.array_equal(views["v"][i].cpu().numpy(), v), f"v of tensor {i}"


def test_keras_adam_eager_bit_for_bit():
    import torch

    from simple_tip_b200 import engine as E

    views, table, p0, grads = _tables(torch, E, np.random.default_rng(0))
    state = torch.zeros(2, dtype=torch.int32, device="cuda")
    for step in grads:
        for view, g in zip(views["g"], step):
            view.copy_(torch.from_numpy(g))
        E.keras_adam(table, len(SIZES), sum(SIZES), state)
    assert state.tolist() == [STEPS, 0]
    _check(views, p0, grads)


def test_keras_adam_graph_replays_bit_for_bit():
    import torch

    from simple_tip_b200 import engine as E

    views, table, p0, grads = _tables(torch, E, np.random.default_rng(1))
    state = torch.zeros(2, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        E.keras_adam(table, len(SIZES), sum(SIZES), state)
    assert state.tolist() == [0, 0]                      # capturing runs nothing
    for step in grads:
        for view, g in zip(views["g"], step):
            view.copy_(torch.from_numpy(g))
        graph.replay()
    assert state.tolist() == [STEPS, 0]
    _check(views, p0, grads)


def test_adam_table_refuses_mismatched_rows():
    import torch

    from simple_tip_b200 import engine as E

    a, b = torch.zeros(4, device="cuda"), torch.zeros(5, device="cuda")
    with pytest.raises(ValueError, match="row 0"):
        E.adam_table([a], [b], [a], [a])
    with pytest.raises(ValueError, match="row 0"):
        E.adam_table([a], [a.double()], [a], [a])


def _xent_reference(z, y):
    z, y = z.astype(np.float64), y.astype(np.float64)
    mx = z.max(axis=1, keepdims=True)
    lse = mx + np.log(np.exp(z - mx).sum(axis=1, keepdims=True))
    logp = z - lse
    loss = float(np.mean(-(y * logp).sum(axis=1)))
    dz = (np.exp(logp) - y) / z.shape[0]
    correct = int(np.sum(z.argmax(axis=1) == y.argmax(axis=1)))
    return loss, dz, correct


@pytest.mark.parametrize("rows, classes", [(128, 10), (32, 2), (1, 10), (77, 10), (1000, 2)])
def test_softmax_xent(rows, classes):
    import torch

    from simple_tip_b200 import engine as E

    rng = np.random.default_rng(rows * 100 + classes)
    z = (rng.normal(size=(rows, classes)) * 3).astype(np.float32)
    labels = rng.integers(0, classes, size=rows)
    y = np.eye(classes, dtype=np.float32)[labels]
    if rows >= 8:
        z[0] = 80.0 * np.sign(rng.normal(size=classes))         # huge logits: a true class far below or far above
        z[1, :] = -80.0
        z[1, labels[1]] = 80.0
        z[2, :] = 80.0
        z[2, labels[2]] = -80.0
        z[3, :2] = z[3].max() + 1.0                            # a tie in z's argmax
        y[4] = 0.0
        y[4, :2] = 0.5                                         # ties in y's argmax
        y[5] = 0.0
        y[5, [0, classes - 1]] = 1.0
    loss = torch.zeros(1, device="cuda")
    correct = torch.zeros(1, dtype=torch.int32, device="cuda")
    dz = torch.empty(rows, classes, device="cuda")
    zt, yt = torch.from_numpy(z).cuda(), torch.from_numpy(y).cuda()
    E.softmax_xent(zt, yt, loss, dz, correct)
    w_loss, w_dz, w_correct = _xent_reference(z, y)
    assert abs(float(loss.item()) - w_loss) <= 1e-6 * abs(w_loss)
    assert np.allclose(dz.cpu().numpy(), w_dz, rtol=1e-6, atol=1e-6 / rows)
    assert int(correct.item()) == w_correct
    loss2 = torch.zeros(1, device="cuda")
    E.softmax_xent(zt, yt, loss2, None, correct)               # no gradient wanted: same loss bits
    assert loss2.item() == loss.item() and int(correct.item()) == w_correct
