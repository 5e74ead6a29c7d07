"""GPU: the device Gaussian-mixture fit (csrc/mixture.cu, engine.gmm_*, core/mixture.py) against NumPy, the float64
reference (oracle/gmm_oracle.py) and live sklearn.  Tolerances come from the fp64 error model of DESIGN.md §5b;
every comparison prints the measured error as a fraction of its bound."""
import os
import warnings

import numpy as np
import pytest

from oracle import gmm_oracle as G

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TWO53 = 2.0 ** 53


def _dev():
    from simple_tip_b200 import engine as E

    return E, E.require_cuda()


def _report(name, err, bound):
    frac = float(np.max(err / bound)) if np.size(err) else 0.0
    print(f"{name}: worst error = {frac:.3g} of the bound")
    return frac


# ---- exact by construction ---------------------------------------------------------------------------------------
EXACT = [  # (d, n, k, dtype, requested scatter chunks)
    (1, 2, 1, np.float32, 0), (2, 3, 3, np.float64, 0), (15, 63, 2, np.float32, 0), (16, 64, 5, np.float64, 0),
    (17, 65, 64, np.float32, 0), (127, 6000, 2, np.float64, 0), (128, 6000, 3, np.float32, 0),
    (128, 6000, 3, np.float64, 1), (128, 6000, 3, np.float32, 7), (129, 100003, 1, np.float64, 0),
    (300, 2000, 64, np.float32, 0), (1024, 6000, 3, np.float64, 0), (2048, 6000, 3, np.float32, 0),
    (2048, 6000, 3, np.float32, 64), (2048, 6000, 1, np.float64, 64)]


def _exact_case(d, n, k, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-8, 9, size=(n, d)).astype(np.float64)
    mu = rng.integers(-2, 3, size=(k, d)).astype(np.float64)
    L = np.triu(rng.integers(-3, 4, size=(k, d, d))).astype(np.float64)
    r8 = rng.integers(0, 9, size=(k, n)).astype(np.float64)          # responsibilities = r8 / 8
    return x, mu, L, r8


@pytest.mark.parametrize("d,n,k,dtype,chunks", EXACT)
def test_exact_passes_equal_numpy_bit_for_bit(d, n, k, dtype, chunks):
    E, dev = _dev()
    x, mu, L, r8 = _exact_case(d, n, k, seed=d * 7 + n + k)
    # every partial is an integer (or a multiple of 1/8) below 2^53, so every summation order is exact
    diff_max = np.abs(x[None] - mu[:, None]).max(axis=(1, 2))                         # per component
    y_bound = diff_max * np.abs(L).sum(axis=1).max(axis=1)                            # |y_ij|
    assert np.all(y_bound ** 2 * d < TWO53)
    assert np.all(8 * diff_max ** 2 * n < TWO53) and 8 * 8 * n < TWO53
    xd = torch.from_numpy(x.astype(dtype)).to(dev)
    mud, Ld = torch.from_numpy(mu).to(dev), torch.from_numpy(L).to(dev)
    resp = torch.from_numpy(r8 / 8).to(dev)
    q = E.gmm_quad(xd, mud, Ld).cpu().numpy()
    want_q = np.stack([np.sum(((x - mu[j]) @ L[j]) ** 2, axis=1) for j in range(k)])
    assert np.array_equal(q, want_q)
    nk, sums, means = E.gmm_moments(xd, resp)
    r = r8 / 8
    want_nk = r.sum(axis=1) + 10 * np.finfo(np.float64).eps
    assert np.array_equal(nk.cpu().numpy(), want_nk)
    assert np.array_equal(sums.cpu().numpy(), r @ x)
    assert np.array_equal(means.cpu().numpy(), (r @ x) / want_nk[:, None])
    used = E.gmm_scatter_chunks(n, d, k, chunks)
    S = E.gmm_scatter(xd, resp, mud, None, 0.0, chunks).cpu().numpy()
    want_S = np.stack([(r[j] * (x - mu[j]).T) @ (x - mu[j]) for j in range(k)])
    assert np.array_equal(S, want_S), f"scatter with {used} chunks"
    if chunks == 64 and d == 2048:
        per_chunk = k * 32 * 33 // 2 * 64 * 64 * 8
        assert used > 1 and used * per_chunk <= 256 << 20 < (used + 1) * per_chunk, used


# ---- one step at a time ------------------------------------------------------------------------------------------
def _data(kind, seed=0, n=4000, d=24, k=3):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(k, d)) * 3.0
    x = centres[rng.integers(0, k, size=n)] + rng.normal(size=(n, d))
    if kind == "dead":
        x = np.maximum(x, 0.0)
        x[:, :3] = 0.0
    return x


def _step_bounds(x, state, ref):
    """DESIGN.md §5b: worst-case error of one device EM step against the float64 reference from the same state."""
    w, mu, prec = state
    n, d = x.shape
    qb = G.quad_bound(x, mu, prec)                                   # [k, n]
    u = G.U
    # a_k = -q/2 + const: |da| <= qb/2 + 4u|a|; resp = exp(a - lse): relative error <= |da_k| + max_j |da_j| + 4u
    q = G.quad(x, mu, prec)
    a = np.abs(G.weighted_log_prob(q, d, w, prec)).T                  # [k, n]
    da = qb / 2 + 4 * u * a
    er = da + da.max(axis=0, keepdims=True) + 4 * u                  # relative error of resp [k, n]
    _, lpn, resp = G.e_step(x, w, mu, prec)
    lb_b = float(np.mean(da.max(axis=0) + 4 * u * np.abs(lpn))) + G.gamma(n) * float(np.mean(np.abs(lpn)))
    r = resp.T                                                       # [k, n]
    nk = r.sum(axis=1)
    g = G.gamma(n + 2)
    w_b = (np.sum(r * er, axis=1) / nk + g) * 2 * ref[1]
    ax = np.abs(x)
    mu_b = ((r * er) @ ax + g * (r @ ax)) / nk[:, None] + (np.sum(r * er, axis=1) / nk + g)[:, None] * np.abs(ref[2])
    cov_b = np.empty_like(ref[3])
    for j in range(len(nk)):
        dd = np.abs(x - ref[2][j])
        m2 = ((r[j] * (er[j] + G.gamma(n + 3))) * dd.T) @ dd / nk[j]
        m1 = (r[j] * dd.T).sum(axis=1) / nk[j]
        cov_b[j] = m2 + np.outer(mu_b[j], m1) + np.outer(m1, mu_b[j]) + (np.sum(r[j] * er[j]) / nk[j] + g) * np.abs(ref[3][j])
    return lb_b, w_b, mu_b, cov_b


def _cond(cov):
    return np.array([np.linalg.cond(c) for c in cov])


@pytest.mark.parametrize("kind", ["blobs", "dead"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_em_step_matches_the_reference_one_step_at_a_time(kind, dtype):
    E, dev = _dev()
    x = _data(kind, seed=1).astype(dtype)
    xh = x.astype(np.float64)
    xd = torch.from_numpy(x).to(dev)
    k = 3
    _, labels, _, _ = E.kmeans_fit(xd, k, 1, 300, 1e-4, 0)
    w, mu, cov, prec = G.initialize(xh, labels.cpu().numpy(), k, 1e-6)
    state = (w, mu, prec)
    for t in range(4):
        ref = G.em_step(xh, w, mu, prec, 1e-6)
        lb, dw, dmu, dcov, dprec = E.gmm_em_step(xd, *(torch.from_numpy(v).to(dev) for v in (w, mu, prec)), 1e-6)
        lb_b, w_b, mu_b, cov_b = _step_bounds(xh, state, ref)
        _report(f"{kind}/{np.dtype(dtype).name} step {t} bound", np.array([abs(lb - ref[0])]), np.array([lb_b]))
        assert abs(lb - ref[0]) <= lb_b
        for name, got, want, b in (("weights", dw, ref[1], w_b), ("means", dmu, ref[2], mu_b),
                                   ("covariances", dcov, ref[3], cov_b)):
            err = np.abs(got.cpu().numpy() - want)
            _report(f"  {name}", err, b + 1e-300)
            assert np.all(err <= b), name
        # the factor: L^T cov L = I to cond(cov) * d * u, and the quadratic forms it produces
        L, C = dprec.cpu().numpy(), dcov.cpu().numpy()
        kap = _cond(C)
        d = x.shape[1]
        for j in range(k):
            eye_err = np.abs(L[j].T @ C[j] @ L[j] - np.eye(d)).max()
            _report(f"  L^T cov L - I [{j}]", np.array([eye_err]), np.array([8 * d * G.U * kap[j]]))
            assert eye_err <= 8 * d * G.U * kap[j]
        q_dev = E.gmm_quad(xd, dmu, dprec).cpu().numpy()
        q_ref = G.quad(xh, ref[2], ref[4])
        qb = (8 * d * G.U * kap[:, None] + 2 * mu_b.max() ) * (q_ref + d) + G.quad_bound(xh, dmu.cpu().numpy(), L)
        _report("  q through the factor", np.abs(q_dev - q_ref), qb)
        assert np.all(np.abs(q_dev - q_ref) <= qb)
        # next step from the DEVICE state, so that errors do not compound
        w, mu, prec = dw.cpu().numpy(), dmu.cpu().numpy(), L
        state = (w, mu, prec)


# ---- whole fits ----------------------------------------------------------------------------------------------------
def _fit_both(x, k, seed=0, max_iter=100, tol=1e-3):
    E, dev = _dev()
    from simple_tip_b200.core.mixture import GaussianMixture

    xd = torch.from_numpy(x).to(dev)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gm = GaussianMixture(k, tol=tol, max_iter=max_iter, random_state=seed).fit(x)
    _, labels, _, _ = E.kmeans_fit(xd, k, 1, 300, 1e-4, seed)
    assert torch.equal(labels, gm.labels_init_), "init labels differ from kmeans_fit(x, K, 1, 300, 1e-4, seed)"
    ref = G.fit(x.astype(np.float64), labels.cpu().numpy(), k, max_iter=max_iter, tol=tol)
    return gm, ref


@pytest.mark.parametrize("kind,seed", [("blobs", 2), ("blobs", 3), ("dead", 4)])
def test_whole_fit_matches_the_reference(kind, seed):
    x = _data(kind, seed=seed)
    gm, ref = _fit_both(x, 3, seed=seed)
    # the stop decision may only differ where the reference's change lies within the bound's reach of tol
    lb_err = 1e-10 * abs(ref["lower_bound"])
    decided = all(m > lb_err for m in ref["margins"])
    if decided:
        assert gm.n_iter_ == ref["n_iter"] and gm.converged_ == ref["converged"]
    else:
        pytest.skip("the reference's stop decision lies within the error bound of tol")
    np.testing.assert_allclose(gm.lower_bounds_, ref["lower_bounds"], rtol=1e-10)
    # final parameters: one step's bound (measured fraction below) times the number of steps
    state = (ref["weights"], ref["means"], ref["prec_chol"])
    again = G.em_step(x, *state, 1e-6)
    _, w_b, mu_b, cov_b = _step_bounds(x, state, again)
    it = gm.n_iter_
    for name, got, want, b in (("weights", gm.weights_, ref["weights"], w_b), ("means", gm.means_, ref["means"], mu_b),
                               ("covariances", gm.covariances_, ref["covariances"], cov_b)):
        err = np.abs(got - want)
        _report(f"{kind} fit {name}", err, it * b + 1e-300)
        assert np.all(err <= it * b), name


def test_live_sklearn_from_the_same_initial_parameters():
    from sklearn.mixture import GaussianMixture as SkGM

    compared = 0
    for kind, seed, rtol in (("blobs", 5, 1e-6), ("dead", 6, None)):
        x = _data(kind, seed=seed)
        gm, ref = _fit_both(x, 3, seed=seed)
        w, mu, cov, _ = ref["init"]
        sk = SkGM(3, weights_init=w, means_init=mu, precisions_init=np.linalg.inv(cov), init_params="random",
                  random_state=0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sk.fit(x)
        if sk.n_iter_ != gm.n_iter_:
            continue                     # the two stop at different iterations: nothing to compare
        compared += 1
        ours, theirs = gm.score_samples(x), sk.score_samples(x)
        if rtol is not None:
            np.testing.assert_allclose(ours, theirs, rtol=rtol)
        else:
            # dead columns: the reference's own spread from sklearn (different factor of the same precision) plus
            # the device's per-step bound on the bound, per row
            ref_s = G.score_samples(x, ref["weights"], ref["means"], ref["prec_chol"])
            b = np.abs(ref_s - theirs) + 1e-6 * np.abs(theirs)
            _report("dead-column score_samples vs sklearn", np.abs(ours - theirs), b)
            assert np.all(np.abs(ours - theirs) <= 2 * b)
    assert compared == 2


def test_mlsa_device_scores_agree_with_its_own_fit():
    from simple_tip_b200.core.surprise import MLSA

    x = _data("blobs", seed=7).astype(np.float32)
    m = MLSA(x, num_components=3, backend="device")
    np.testing.assert_allclose(m(x[:500]), -m.gmm.score_samples(x[:500]), rtol=1e-4)


def test_two_fits_give_identical_bits():
    from simple_tip_b200.core.mixture import GaussianMixture

    x = _data("dead", seed=8).astype(np.float32)
    a = GaussianMixture(3).fit(x)
    b = GaussianMixture(3).fit(x)
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert a.lower_bounds_ == b.lower_bounds_ and a.n_iter_ == b.n_iter_


def test_non_positive_definite_covariance_raises_sklearns_error():
    E, dev = _dev()
    cov = torch.tensor([[[2.0, 0.0], [0.0, 1.0]], [[1.0, 2.0], [2.0, 1.0]]], dtype=torch.float64, device=dev)
    _, _, info = E.gmm_factor(cov)
    assert info.cpu().tolist()[0] == 0 and info.cpu().tolist()[1] != 0
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        E._raise_if_failed(info)
    torch.cuda.synchronize()             # no kernel fault


# ---- integration -----------------------------------------------------------------------------------------------------
def test_mlsa_plausability_on_the_device():
    from simple_tip_b200.core.surprise import MLSA

    rng = np.random.RandomState(42)
    activations = np.concatenate([rng.random((10000, 10)), rng.random((10000, 10)) + 0.4,
                                  rng.random((10000, 10)) + 0.9])
    mlsa = MLSA(activations, num_components=3, backend="device")
    test_activations = np.array([[0.5] * 10, [0.9] * 10, [1.4] * 10])
    assert len(set(mlsa.gmm.predict(test_activations))) == 3
    assert np.all(mlsa(test_activations + 2) > mlsa(test_activations))


def test_pc_mlsa_through_the_environment_variable(monkeypatch):
    from sklearn.mixture import GaussianMixture as SkGM

    from simple_tip_b200.core.surprise import MLSA, MultiModalSA

    rng = np.random.default_rng(9)
    x = np.concatenate([_data("blobs", seed=10 + c, n=1500, d=16) + 5 * c for c in range(3)]).astype(np.float32)
    y = np.repeat(np.arange(3), 1500)
    monkeypatch.setenv("B200TIP_GMM", "device")
    sa = MultiModalSA.build_by_class(x, y, lambda x, y: MLSA(x, num_components=3))
    test = x[rng.choice(len(x), 300, replace=False)]
    pred = y[rng.choice(len(x), 300, replace=False)]
    got = sa(test, pred)
    for c, m in sa.modal_sa.items():
        assert m.backend == "device"
        w, mu, cov, _ = G.initialize(x[y == c].astype(np.float64), m.gmm.labels_init_.cpu().numpy(), 3, 1e-6)
        sk = SkGM(3, weights_init=w, means_init=mu, precisions_init=np.linalg.inv(cov), init_params="random",
                  random_state=0).fit(x[y == c])
        if sk.n_iter_ != m.gmm.n_iter_:
            continue
        rows = pred == c
        np.testing.assert_allclose(got[rows], -sk.score_samples(test[rows]), rtol=1e-4)


def test_cuda_tensor_input_gives_the_same_bits():
    E, dev = _dev()
    from simple_tip_b200.core.mixture import GaussianMixture

    x = _data("blobs", seed=12).astype(np.float32)
    a = GaussianMixture(3).fit(x)
    xt = torch.from_numpy(x).to(dev)
    b = GaussianMixture(3).fit(xt)
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert np.array_equal(a.score_samples(x), b.score_samples(xt).cpu().numpy())
