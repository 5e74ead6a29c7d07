"""oracle/train_oracle.py without a GPU: the float64 cross-entropy against torch's float64 autograd, a float32
restatement of the xent kernel's order inside the derived bounds and its naive-route mutants outside them, and the
float32 Adam restatement inside its bound of Keras' float64 Adam with torch's epsilon placement outside it."""
import numpy as np
import pytest
import torch

from oracle import train_oracle as T

F = np.float32


def _tree(x):
    """The kernel's 5-level xor-shuffle tree over 32 lanes (zero-padded), in float32: [R, C] -> [R]."""
    x = np.concatenate([x.astype(F), np.zeros((x.shape[0], 32 - x.shape[1]), F)], axis=1)
    for o in (16, 8, 4, 2, 1):
        x = (x[:, :o] + x[:, o:2 * o]).astype(F)
    return x[:, 0]


def _xent_f32(z, y, naive_grad=False, naive_loss=False):
    """tip_softmax_xent's routes in NumPy float32, row by row (np.exp / np.log standing in for CUDA's expf / logf):
    (row loss [R], dz [R, C] before the division by the row count).  naive_grad: p - 1 for y = 1 instead of -o / s;
    naive_loss: logf(s) at a lane of the max instead of log1pf(o)."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        mx = z.max(axis=1, keepdims=True)
        e = np.exp((z - mx).astype(F)).astype(F)
        s = _tree(e)[:, None]
        o = np.stack([_tree(np.where(np.arange(z.shape[1]) == k, F(0), e)) for k in range(z.shape[1])], axis=1)
        top = z == mx
        log_s = np.log(s).astype(F)
        nlp = np.where(top, log_s if naive_loss else np.log1p(o), ((mx - z).astype(F) + log_s).astype(F)).astype(F)
        loss = _tree(np.where(y != 0, (y * nlp).astype(F), F(0)))
        true_route = (e / s - F(1)).astype(F) if naive_grad else -(o / s).astype(F)
        dz = np.where(y == 1, true_route, (e / s).astype(F) - y).astype(F)
    return loss.astype(np.float64), dz.astype(np.float64)


def _violations(z, y, loss, dz):
    ref = T.xent_reference(z, y)
    lb, db = T.xent_bounds(z, y, ref)
    inf = np.isinf(ref.loss)
    with np.errstate(invalid="ignore"):
        bad_loss = np.where(inf, loss != ref.loss, ~(np.abs(loss - ref.loss) <= lb))
    return bad_loss, ~(np.abs(dz - ref.dz) <= db)


@pytest.mark.parametrize("targets", ["one-hot", "soft", "zero"])
@pytest.mark.parametrize("classes", [1, 2, 10, 32])
def test_xent_reference_equals_torch_autograd(targets, classes):
    rng = np.random.default_rng(classes)
    z = (rng.normal(size=(64, classes)) * 4).astype(F)
    y = {"one-hot": np.eye(classes, dtype=F)[rng.integers(0, classes, 64)],
         "soft": rng.dirichlet(np.ones(classes), size=64).astype(F),
         "zero": np.zeros((64, classes), F)}[targets]
    ref = T.xent_reference(z, y)
    zt = torch.from_numpy(z).double().requires_grad_()
    yt = torch.from_numpy(y).double()
    loss = torch.nn.functional.cross_entropy(zt, yt, reduction="none")
    loss.sum().backward()
    np.testing.assert_allclose(ref.loss, loss.detach().numpy(), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(ref.nlp, -torch.log_softmax(zt, dim=1).detach().numpy(), rtol=1e-13, atol=1e-15)
    # autograd gives p * sum(y) - y, the reference p - y: equal where the targets sum to 1
    want = zt.grad.numpy() + ref.p * (1 - y.astype(np.float64).sum(axis=1, keepdims=True))
    np.testing.assert_allclose(ref.dz, want, rtol=1e-12, atol=1e-15)
    assert np.array_equal(ref.argmax_z, z.argmax(axis=1)) and np.array_equal(ref.argmax_y, y.argmax(axis=1))


def test_xent_reference_keeps_the_confident_rows_precision():
    z = np.array([[40.0, 0.0, 0.0], [17.0, 0.0, -np.inf], [3.0, 3.0, 0.0]], F)
    y = np.array([[1, 0, 0], [1, 0, 1], [0.5, 0.5, 0]], F)
    ref = T.xent_reference(z, y)
    assert ref.nlp[0, 0] == pytest.approx(2 * np.exp(-40.0), rel=1e-15)
    assert ref.dz[0, 0] == pytest.approx(-2 * np.exp(-40.0) / (1 + 2 * np.exp(-40.0)), rel=1e-15)
    assert ref.loss[1] == np.inf and ref.dz[1, 2] == -1.0
    assert ref.argmax_z[2] == 0 and ref.argmax_y[2] == 0


@pytest.mark.parametrize("classes", [1, 2, 3, 10, 31, 32])
def test_the_kernels_routes_in_float32_stay_inside_the_bounds(classes):
    z, y = T.xent_bank(np.random.default_rng(classes), 960, classes)
    bad_loss, bad_dz = _violations(z, y, *_xent_f32(z, y))
    assert not bad_loss.any(), np.flatnonzero(bad_loss)[:10]
    assert not bad_dz.any(), np.argwhere(bad_dz)[:10]


@pytest.mark.parametrize("classes", [2, 10, 32])
def test_the_naive_routes_fail_the_bounds_at_margins_of_17_and_more(classes):
    """p - 1 for the true class's gradient and logf(s) for the max lane's loss lose the relative precision the
    bounds ask for once the true class leads by 17 or more: always where o < 2^-24 (s rounds to 1), and on all but
    a stray row elsewhere."""
    rng = np.random.default_rng(17 + classes)
    n = 400
    label = rng.integers(0, classes, n)
    z = rng.normal(size=(n, classes))
    z[np.arange(n), label] = np.max(z, axis=1) + rng.uniform(17, 40, n)
    z = z.astype(F)
    y = np.eye(classes, dtype=F)[label]
    ok_loss, ok_dz = _violations(z, y, *_xent_f32(z, y))
    assert not ok_loss.any() and not ok_dz.any()
    ref = T.xent_reference(z, y)
    certain = -ref.dz[np.arange(n), label] < 2.0 ** -24
    assert certain.sum() >= n // 4
    bad_loss = _violations(z, y, *_xent_f32(z, y, naive_loss=True))[0]
    bad_dz = _violations(z, y, *_xent_f32(z, y, naive_grad=True))[1][np.arange(n), label]
    for bad in (bad_loss, bad_dz):
        assert bad[certain].all() and bad.mean() >= 0.99, (bad.mean(), np.flatnonzero(~bad)[:10])


def _adam_case(rng, n, steps, scales):
    p = rng.normal(size=n).astype(F)
    scale = np.asarray(scales, dtype=np.float64)[np.arange(n) % len(scales)]
    grads = [(rng.normal(size=n) * scale).astype(F) for _ in range(steps)]
    return p, grads


@pytest.mark.parametrize("t0, hyper", [(0, {}), (999, {}), (0, dict(lr=3e-2, beta1=0.0, epsilon=1e-3)),
                                       (5, dict(lr=1e-4, beta1=0.5, beta2=0.99, epsilon=1e-8))])
def test_adam_restatement_within_its_bound_of_keras_f64(t0, hyper):
    rng = np.random.default_rng(t0 + len(hyper))
    p, grads = _adam_case(rng, 5000, 50, [1e-9, 1e-7, 1e-5, 1e-3, 1e-1, 1.0, 10.0, 1e3])
    m0 = v0 = None
    if t0:
        m0 = (rng.normal(size=p.size) * 1e-2).astype(F)
        v0 = (rng.random(p.size) * 1e-4).astype(F)
    got = T.adam_restatement(p, grads, t0, m=m0, v=v0, **hyper)
    want = T.keras_adam_f64(p, grads, t0, m=m0, v=v0, **hyper)
    bounds = T.keras_adam_bound(p, grads, t0, m=m0, v=v0, **hyper)
    for name, a, b, bound in zip("pmv", got, want, bounds):
        err = np.abs(a.astype(np.float64) - b)
        assert np.all(err <= bound), (name, float(np.max(err / np.maximum(bound, 1e-300))))


def test_torch_adam_lies_outside_the_bound_on_tiny_gradients():
    """With |g| ~ 1e-9..1e-7, sqrt(v) << epsilon, where Keras' step lr sqrt(1 - b2^t) m / ((1 - b1^t) eps) and
    torch's lr m / ((1 - b1^t) eps) differ by the factor sqrt(1 - b2^t): a bound that let torch's form pass could not
    tell the two apart on the GPU."""
    rng = np.random.default_rng(3)
    n = 4000
    sign = rng.choice([-1.0, 1.0], size=n)
    p = rng.normal(size=n).astype(F)
    grads = [(sign * 10.0 ** rng.uniform(-9, -7, size=n)).astype(F) for _ in range(50)]
    keras = T.keras_adam_f64(p, grads)[0]
    bound = T.keras_adam_bound(p, grads)[0]
    assert np.all(np.abs(T.adam_restatement(p, grads)[0] - keras) <= bound)
    assert np.all(np.abs(T.torch_adam_f64(p, grads)[0] - keras) > bound)


def test_gather_reference_rounds_to_nearest_even():
    pool = np.array([[1 + 2.0 ** -24], [1 + 3 * 2.0 ** -24], [2.0 ** 128 - 2.0 ** 103], [-1e39], [2.0 ** -150],
                     [3 * 2.0 ** -150], [-0.0]])
    rows = np.arange(7)[None, :]
    got = T.gather_reference(pool, rows, rows, 0, 7, False)[0, :, 0]
    assert got.dtype == F
    assert got.tolist()[:2] == [1.0, 1 + 2.0 ** -22]
    assert got[2] == np.inf and got[3] == -np.inf and got[4] == 0.0 and got[5] == F(2.0 ** -148)
    assert np.signbit(got[6])
