"""The training kernels against float64 references (oracle/train_oracle.py).

tip_softmax_xent_seg, row by row: with one row per segment each row's loss comes back on its own, so the bound
applies to every row, not only to a batch mean.  The bounds are derived in `train_oracle.xent_bounds` from the
kernel's operation order, u = 2^-24 and D the p-weighted mean of max(z) - z_c over the lanes below the max:
  * loss of a row: (32 + 2 D) u sum_c y_c (-log p_c) + 32 * 2^-126 (the float32 underflow);
  * dz: u ((32 + 2 D) mag + 2 p_c d_c) + 8 * 2^-149, mag = |p - y| where y_c = 1 (the -o / s route) and p + y
    elsewhere; both divided by the row count for a segment of several rows, whose mean loss adds u |mean|;
  * correct: exact, first-index argmax of z and of y.
Logits reach +-1e30 but not +-3e38, where mx - z overflows in float32 and not in float64.  The naive routes (p - 1,
logf(s)) fail these bounds at margins of 17 and more (tests/test_train_oracle.py).

tip_keras_adam: bit for bit against `adam_restatement` at the table's edges, eagerly and replayed from a graph, and
within `keras_adam_bound` of Keras' float64 Adam over 50 steps (the bound torch's epsilon placement fails).

tip_stack_gather: bit patterns equal to `gather_reference` at the float64 -> float32 rounding's edges.

training.evaluate / evaluate_stack: exact accuracies and losses within the per-row bound, on the logits the networks
themselves produce in those calls."""
import numpy as np
import pytest

from oracle import train_oracle as T

pytestmark = pytest.mark.gpu

F = np.float32
U = 2.0 ** -24


def _cuda(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run_xent(z, y, segments, dz=True):
    """tip_softmax_xent_seg on z, y [segments * rows, C]: (loss [segments], dz [segments * rows, C], correct)."""
    import torch

    from simple_tip_b200 import engine as E

    rows = z.shape[0] // segments
    zt, yt = _cuda(z).view(segments, rows, -1), _cuda(y).view(segments, rows, -1)
    loss = torch.full((segments,), -7.0, device="cuda")
    correct = torch.full((segments,), -7, dtype=torch.int32, device="cuda")
    dzt = torch.full_like(zt, np.nan) if dz else None
    E.softmax_xent_seg(zt, yt, loss, dzt, correct)
    return (loss.cpu().numpy().astype(np.float64), dzt.cpu().numpy().reshape(z.shape).astype(np.float64) if dz else None,
            correct.cpu().numpy())


def _check_xent(z, y, segments, loss, dz, correct):
    rows = z.shape[0] // segments
    ref = T.xent_reference(z, y)
    lb, db = T.xent_bounds(z, y, ref)
    want = ref.loss.reshape(segments, rows)
    inf = np.isinf(want).any(axis=1)
    mean = np.where(inf[:, None], 0.0, want).mean(axis=1)
    bound = lb.reshape(segments, rows).sum(axis=1) / rows + U * np.abs(mean)
    assert np.array_equal(loss[inf], np.full(inf.sum(), np.inf)), "a -inf logit under a target gives +inf"
    err = np.abs(loss[~inf] - mean[~inf])
    assert np.all(err <= bound[~inf]), ("loss", np.argmax(err / bound[~inf]), float(np.max(err / bound[~inf])))
    if dz is not None:
        derr = np.abs(dz - ref.dz / rows)
        dbound = db / rows + 2.0 ** -150
        assert np.all(derr <= dbound), ("dz", np.unravel_index(np.argmax(derr / dbound), dz.shape),
                                        float(np.max(derr / dbound)))
    hit = (ref.argmax_z == ref.argmax_y).reshape(segments, rows).sum(axis=1)
    assert np.array_equal(correct, hit), "correct counts differ"


@pytest.mark.parametrize("classes", range(1, 33))
def test_xent_row_by_row_on_70000_segments(classes):
    """One row per segment: every row's loss on its own, over 70 000 segments (gridDim.x above 65 535)."""
    z, y = T.xent_bank(np.random.default_rng(classes), 4800, classes)
    z, y = np.resize(z, (70_000, classes)), np.resize(y, (70_000, classes))
    _check_xent(z, y, 70_000, *_run_xent(z, y, 70_000))


@pytest.mark.parametrize("segments", [1, 7])
@pytest.mark.parametrize("rows", [1, 31, 32, 33, 1023, 1025])
def test_xent_multi_row_segments(rows, segments):
    rng = np.random.default_rng(rows * 10 + segments)
    for classes in range(1, 33):
        z, y = T.xent_bank(rng, rows * segments, classes, inf_targets=False)
        _check_xent(z, y, segments, *_run_xent(z, y, segments))
        loss, _, correct = _run_xent(z, y, segments, dz=False)
        _check_xent(z, y, segments, loss, None, correct)


@pytest.mark.parametrize("classes", [10, 32])
def test_xent_one_segment_of_300000_rows(classes):
    """Each warp sums 9 375 row losses in double."""
    z, y = T.xent_bank(np.random.default_rng(classes), 4800, classes, inf_targets=False)
    z, y = np.resize(z, (300_000, classes)), np.resize(y, (300_000, classes))
    _check_xent(z, y, 1, *_run_xent(z, y, 1))


def test_xent_infinite_rows_stay_in_their_segment():
    z, y = T.xent_bank(np.random.default_rng(5), 7 * 48, 10)
    loss, dz, correct = _run_xent(z, y, 7)
    _check_xent(z, y, 7, loss, dz, correct)
    assert np.isinf(loss).any() and np.isfinite(dz).all()


# ---- tip_keras_adam ------------------------------------------------------------------------------------------------------
HYPER = {"default": {}, "beta1=0": dict(lr=3e-2, beta1=0.0, epsilon=1e-3),
         "other": dict(lr=2.5e-4, beta1=0.5, beta2=0.99, epsilon=1e-8)}


def _layout(rng):
    """256 tensors: (numel, the float offsets of param, grad, m and v in their buffers, mod 4 = their alignment)."""
    spec = []
    for n in range(1, 8):
        for a in range(4):                                   # head lengths 3, 2, 1, 0 (a = 1, 2, 3, 0)
            spec.append((n, (a,) * 4))
    for role in range(4):                                    # one array misaligned against the other three
        for n in (5, 9, 33, 1000):
            spec.append((n, tuple(1 if r == role else 0 for r in range(4))))
    spec += [(4097, (0,) * 4), (100_003, (2,) * 4), (70_001, (1, 2, 3, 0))]
    while len(spec) < 253:
        spec.append((int(rng.integers(1, 300)), tuple(int(k) for k in rng.integers(0, 4, 4))))
    spec = [(0, (0,) * 4)] + spec[:127] + [(0, (1,) * 4)] + spec[127:] + [(0, (3,) * 4)]
    assert len(spec) == 256
    return spec


def _grad(rng, n, step, k):
    """Per element one of: 0, +-1e-40 (subnormal), +-1e-9, normal, +-1e3, +-2e19 (g * g overflows) and NaN."""
    kinds = (np.arange(n) + step + k) % 7
    mag = np.array([0.0, 1e-40, 1e-9, 1.0, 1e3, 2e19, np.nan])[kinds]
    return (mag * rng.normal(size=n)).astype(F)


def _same_bits(a, b):
    a, b = np.asarray(a, F), np.asarray(b, F)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("hyper", list(HYPER))
@pytest.mark.parametrize("t0", [0, 1, 999, 2 ** 20])
def test_keras_adam_bit_for_bit_at_the_edges(t0, hyper, graph):
    import torch

    from simple_tip_b200 import engine as E

    rng = np.random.default_rng(t0 + 10 * len(hyper) + graph)
    spec = _layout(rng)
    steps = 3
    starts = np.cumsum([0] + [(n + 11) // 4 * 4 for n, _ in spec])   # multiples of 4: a tensor's offsets set its alignment
    bufs = [torch.zeros(int(starts[-1]), device="cuda") for _ in range(4)]
    views = [[b[s + offs[r]:s + offs[r] + n] for (n, offs), s in zip(spec, starts.tolist())] for r, b in enumerate(bufs)]
    p0 = [rng.normal(size=n).astype(F) for n, _ in spec]
    m0 = [(rng.normal(size=n) * 1e-2).astype(F) if t0 else np.zeros(n, F) for n, _ in spec]
    v0 = [(rng.random(n) * 1e-3).astype(F) if t0 else np.zeros(n, F) for n, _ in spec]
    for r, init in ((0, p0), (2, m0), (3, v0)):
        for view, a in zip(views[r], init):
            view.copy_(torch.from_numpy(a))
    grads = [[_grad(rng, n, s, k) for k, (n, _) in enumerate(spec)] for s in range(steps)]
    table = E.adam_table(*views)
    total = sum(n for n, _ in spec)
    state = torch.tensor([t0, 0], dtype=torch.int32, device="cuda")
    kw = HYPER[hyper]
    if graph:
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            E.keras_adam(table, len(spec), total, state, **kw)
        assert state.tolist() == [t0, 0]
    for s in range(steps):
        for view, gr in zip(views[1], grads[s]):
            view.copy_(torch.from_numpy(gr))
        if graph:
            g.replay()
        else:
            E.keras_adam(table, len(spec), total, state, **kw)
        assert state.tolist() == [t0 + s + 1, 0]
    for k, (n, offs) in enumerate(spec):
        want = T.adam_restatement(p0[k], [gr[k] for gr in grads], t0, m=m0[k], v=v0[k], **kw)
        for r, name, w in zip((0, 2, 3), "pmv", want):
            assert _same_bits(views[r][k].cpu().numpy(), w), (name, k, n, offs)


def test_keras_adam_within_its_bound_of_keras_f64():
    import torch

    from simple_tip_b200 import engine as E

    rng = np.random.default_rng(50)
    scales = [1e-9, 1e-7, 1e-5, 1e-3, 1e-1, 1.0, 10.0, 1e3]
    sizes = [1, 7, 4096, 33_333, 5]
    p0 = [rng.normal(size=n).astype(F) for n in sizes]
    tensors = [[_cuda(a.copy()) for a in p0]] + [[torch.zeros(n, device="cuda") for n in sizes] for _ in range(3)]
    table = E.adam_table(*tensors)
    state = torch.zeros(2, dtype=torch.int32, device="cuda")
    signs = [rng.choice([-1.0, 1.0], size=n) for n in sizes]          # fixed per element: m does not cancel
    grads = [[(s * np.abs(rng.normal(size=n)) * np.array(scales)[np.arange(n) % len(scales)]).astype(F)
              for n, s in zip(sizes, signs)] for _ in range(50)]
    for step in grads:
        for t, g in zip(tensors[1], step):
            t.copy_(torch.from_numpy(g))
        E.keras_adam(table, len(sizes), sum(sizes), state)
    assert state.tolist() == [50, 0]
    for k in range(len(sizes)):
        gk = [g[k] for g in grads]
        want, bound = T.keras_adam_f64(p0[k], gk), T.keras_adam_bound(p0[k], gk)
        for name, t, w, b in zip("pmv", (tensors[0][k], tensors[2][k], tensors[3][k]), want, bound):
            err = np.abs(t.cpu().numpy().astype(np.float64) - w)
            assert np.all(err <= b), (name, k, float(np.max(err / b)))
        # the bound tells Keras' epsilon from torch's where |g| <= 1e-7 (sqrt(v) << epsilon)
        tiny = np.arange(sizes[k]) % len(scales) < 2
        assert np.all(np.abs(T.torch_adam_f64(p0[k], gk)[0] - want[0])[tiny] > bound[0][tiny]), k


# ---- tip_stack_gather --------------------------------------------------------------------------------------------------
def _special_f64(rng, n):
    """float64 values at the edges of the rounding to float32, then normal values to fill n."""
    f = rng.normal(size=64).astype(F)
    mids = (f.astype(np.float64) + np.nextafter(f, np.inf).astype(np.float64)) / 2      # ties: to even
    fmax = float(np.finfo(F).max)
    edge = [fmax * (1 + 2.0 ** -25), -fmax * (1 + 2.0 ** -25), 2.0 ** 128 - 2.0 ** 103, -(2.0 ** 128 - 2.0 ** 103),
            1e39, -1e39, np.inf, -np.inf, 1e-40, -1e-40, 2.0 ** -150, 3 * 2.0 ** -150, -3 * 2.0 ** -150,
            2.0 ** -151, -(2.0 ** -151), 2.0 ** -150 * (1 + 2.0 ** -20), np.nan, -0.0, 0.0, 1 + 2.0 ** -24,
            1 + 3 * 2.0 ** -24, 2.0 ** -126 * (1 - 2.0 ** -25)]
    vals = np.concatenate([mids, edge])
    return np.resize(np.concatenate([vals, rng.normal(size=max(n - vals.size, 0)) * 3]), n)


def _gather_bits(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype
    if want.dtype == np.int32:
        return np.array_equal(got, want)
    nan = np.isnan(want)                       # the NaN payload is not specified, only that it stays NaN
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


@pytest.mark.parametrize("m", [1, 2, 80, 300])
@pytest.mark.parametrize("dtype", ["float64", "float32", "int32"])
def test_stack_gather_bits_equal_the_reference(m, dtype):
    import torch

    from simple_tip_b200 import engine as E

    rng = np.random.default_rng(m)
    n_pool, n_rows, n_perm = 40, 57, 50                     # repeated pool rows; n_perm < n_rows
    rows = rng.integers(0, n_pool, size=(m, n_rows))
    perm = np.stack([rng.permutation(n_perm) for _ in range(m)])
    shapes = [((1,), False), ((1, 1, 1), True), ((1, 1, 3), True), ((1, 1, 7), True), ((2, 3, 5), True),
              ((13,), False)]
    for shape, interleave in shapes:
        elems = int(np.prod(shape))
        if dtype == "int32":
            flat = rng.integers(-2 ** 31, 2 ** 31, size=n_pool * elems, dtype=np.int64)
            flat[:2] = [-2 ** 31, 2 ** 31 - 1]
            pool = rng.permutation(flat).astype(np.int32)
        elif dtype == "float64":
            pool = rng.permutation(_special_f64(rng, n_pool * elems))
        else:
            with np.errstate(over="ignore"):
                pool = rng.permutation(_special_f64(rng, n_pool * elems).astype(F))
        pool = pool.reshape(n_pool, *shape)
        for interleaved in ((False, True) if interleave else (False,)):
            for b in (1, n_perm):
                start = n_perm - b
                got = E.stack_gather(_cuda(pool), _cuda(rows), _cuda(perm), start, b, interleaved)
                want = T.gather_reference(pool, rows, perm, start, b, interleaved)
                assert _gather_bits(got.cpu().numpy(), want), (shape, interleaved, b)


@pytest.fixture
def no_launch(monkeypatch):
    from simple_tip_b200 import _lib

    before = _lib.launch_count()

    def refuse():
        raise AssertionError("the wrapper reached the library")

    monkeypatch.setattr(_lib, "load", refuse)
    yield
    monkeypatch.undo()
    assert _lib.launch_count() == before


def test_stack_gather_refuses_perm_outside_the_rows_and_host_tables(no_launch):
    import torch

    from simple_tip_b200 import engine as E

    pool = torch.zeros((10, 3), device="cuda")
    rows = torch.zeros((2, 4), dtype=torch.int64, device="cuda")
    perm = torch.arange(3, device="cuda").expand(2, 3).contiguous()
    for bad in (4, -1, 2 ** 40):
        p = perm.clone()
        p[1, 2] = bad
        with pytest.raises(ValueError, match="perm index"):
            E.stack_gather(pool, rows, p, 0, 3)
    with pytest.raises(ValueError, match="pool's device"):
        E.stack_gather(pool, rows.cpu(), perm, 0, 3, check=False)
    with pytest.raises(ValueError, match="pool's device"):
        E.stack_gather(pool, rows, perm.cpu(), 0, 3, check=False)


def test_xent_wrappers_refuse_tensors_off_zs_device(no_launch):
    import torch

    from simple_tip_b200 import engine as E

    z, y = torch.zeros(4, 3, device="cuda"), torch.zeros(4, 3, device="cuda")
    loss, correct, dz = torch.zeros(1, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros_like(z)
    for i in range(4):
        args = [y, loss, dz, correct]
        args[i] = args[i].cpu()
        with pytest.raises(ValueError, match="one CUDA device"):
            E.softmax_xent(z, *args)
        with pytest.raises(ValueError, match="one CUDA device"):
            E.softmax_xent_seg(z[None], args[0][None], args[1], args[2][None], args[3])


# ---- evaluation ----------------------------------------------------------------------------------------------------------
def _spy(obj, record):
    inner = obj.logits

    def logits(x):
        z = inner(x)
        record.append(z.detach().cpu().numpy().copy())
        return z
    obj.logits = logits


def _data(torch, name, n, rng):
    if name == "imdb":
        x = rng.integers(1, 2000, size=(n, 100)).astype(np.int32)
        x[:, :40] = 0
        classes = 2
    else:
        x, classes = rng.random((n, 28, 28, 1)).astype(F), 10
    y = np.eye(classes, dtype=F)[rng.integers(0, classes, n)]
    return _cuda(x), _cuda(y), y


def _check_eval(loss, acc, z, y):
    ref = T.xent_reference(z, y)
    lb, _ = T.xent_bounds(z, y, ref)
    n = y.shape[0]
    assert acc == int(np.sum(ref.argmax_z == ref.argmax_y)) / n
    want = float(np.mean(ref.loss))
    assert abs(loss - want) <= lb.sum() / n + 2 * U * want, (loss, want)


@pytest.mark.parametrize("n, batch", [(1000, 384), (5, 1), (1, 64)])
@pytest.mark.parametrize("name", ["mnist", "imdb"])
def test_evaluate_against_the_reference_on_its_own_logits(name, n, batch):
    import torch

    from simple_tip_b200.case_studies import CASE_STUDIES
    from simple_tip_b200.core import training

    torch.manual_seed(n + batch)
    model = CASE_STUDIES[name].network().cuda()
    x, yt, y = _data(torch, name, n, np.random.default_rng(n))
    record = []
    _spy(model, record)
    loss, acc = training.evaluate(model, x, yt, rows=batch)
    z = np.concatenate(record)
    assert z.shape == y.shape
    _check_eval(loss, acc, z, y)


@pytest.mark.parametrize("n, batch", [(1000, 384), (5, 1), (1, 64)])
@pytest.mark.parametrize("name", ["mnist", "imdb"])
def test_evaluate_stack_against_the_reference_on_its_own_logits(name, n, batch):
    import torch

    from simple_tip_b200.case_studies import CASE_STUDIES
    from simple_tip_b200.case_studies.stacked import stack
    from simple_tip_b200.core import training

    torch.manual_seed(n + batch)
    m = 3
    net = stack([CASE_STUDIES[name].network() for _ in range(m)]).cuda()
    rng = np.random.default_rng(n + 1)
    x, yt, y = _data(torch, name, 2 * n + 3, rng)
    rows = np.stack([rng.permutation(2 * n + 3)[:n] for _ in range(m)])
    record = []
    _spy(net, record)
    losses, accs = training.evaluate_stack(net, x, yt, _cuda(rows), batch)
    z = np.concatenate(record, axis=1)
    assert z.shape == (m, n, y.shape[1])
    for k in range(m):
        _check_eval(losses[k], accs[k], z[k], y[rows[k]])
