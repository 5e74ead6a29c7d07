"""GPU: LSA's device fit (tip_col_var, tip_whiten_dmma, engine.kde_fit, StableGaussianKDE.from_device,
LSA(backend="device")) against NumPy, the host fit and the float64 restatement of oracle/kdefit_oracle.py.  Bounds
come from DESIGN.md §5d; every bounded comparison prints the measured error as a fraction of its bound."""
import warnings

import numpy as np
import pytest

from oracle import kdefit_oracle as K

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

LSA_RTOL, LSA_ATOL = 1e-4, 2e-4          # the LSA tolerance of the existing parity tests


def _dev():
    from simple_tip_b200 import engine as E

    return E, E.require_cuda()


def _report(name, err, bound):
    frac = float(np.max(np.asarray(err) / np.asarray(bound), initial=0.0))
    print(f"{name}: worst error = {frac:.3g} of the bound")
    return frac


def _lsa(x, **kw):
    from simple_tip_b200.core.surprise import LSA

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return LSA(x, **kw)


def _close(got, want):
    assert np.array_equal(np.isinf(got), np.isinf(want))
    f = np.isfinite(want)
    np.testing.assert_allclose(got[f], want[f], rtol=LSA_RTOL, atol=LSA_ATOL)


@pytest.fixture(scope="module")
def relu():
    """60 000 x 2304 ReLU-like float32 traces; column 0 dead, 1 constant, 2 at a large offset, 3 ~ a 1e4 offset."""
    rng = np.random.default_rng(5)
    x = np.maximum(rng.normal(size=(60000, 2304)).astype(np.float32) * rng.uniform(0.1, 3, 2304).astype(np.float32)
                   + rng.normal(size=2304).astype(np.float32), 0)
    x[:, 0] = 0
    x[:, 1] = 3.7
    x[:, 2] = 1e4 + rng.normal(size=60000).astype(np.float32)
    x[:, 3] = 3e5 + np.float32(0.25) * rng.integers(0, 9, 60000).astype(np.float32)
    return x


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 3, 300, 1600, 2304])
@pytest.mark.parametrize("n", [1, 2, 7, 6000, 60000])
def test_col_var_is_np_var_bit_for_bit(relu, n, d, dtype):
    E, dev = _dev()
    for first in ((0, 2) if d == 1 else (0,)):           # d = 1: the dead column and the offset one
        x = np.ascontiguousarray(relu[:n, first:first + d]).astype(dtype)
        var, mean, flags = E.col_var(torch.from_numpy(x).to(dev))
        want = np.var(x, axis=0)
        assert var.dtype == torch.from_numpy(x).dtype
        assert np.array_equal(var.cpu().numpy(), want), np.flatnonzero(var.cpu().numpy() != want)[:5]
        assert np.array_equal(mean.cpu().numpy(), x.astype(np.float64).mean(axis=0))
        assert int(flags.item()) == 0


def test_oracle_fma_defect_is_visible_on_the_offset_columns(relu):
    x = np.ascontiguousarray(relu[:6000, :8])
    assert not np.array_equal(K.var(x, fma=True), np.var(x, axis=0))


@pytest.mark.parametrize("max_features", [300, 30])
def test_ties_at_the_selection_boundary_give_the_hosts_removed_neurons(max_features):
    rng = np.random.default_rng(max_features)
    base = np.maximum(rng.normal(size=(2000, 200)).astype(np.float32), 0)
    x = np.ascontiguousarray(np.concatenate([base, base[:, ::-1], base[:, :40]], axis=1))   # every column duplicated
    host = _lsa(x, max_features=max_features)
    dev = _lsa(x, max_features=max_features, backend="device")
    assert host.removed_neurons == dev.removed_neurons
    assert host.kde.prepare_failed == dev.kde.prepare_failed


def test_var_threshold_gives_the_hosts_set():
    x = np.maximum(np.random.default_rng(2).normal(size=(3000, 60)) * np.linspace(0.1, 2, 60), 0).astype(np.float32)
    host = _lsa(x, var_threshold=0.3, max_features=None)
    dev = _lsa(x, var_threshold=0.3, max_features=None, backend="device")
    assert np.array_equal(host.removed_neurons, dev.removed_neurons) and len(host.removed_neurons) > 0
    probe = x[:50] * 1.1
    np.testing.assert_allclose(dev(probe), host(probe), rtol=LSA_RTOL, atol=LSA_ATOL)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d_kept", [1, 17, 300])
def test_scatter_is_np_cov_bit_for_bit_through_the_column_gather(d_kept, dtype):
    E, dev = _dev()
    n, width = 1024, 460
    rng = np.random.default_rng(d_kept)
    x = rng.integers(-8, 9, size=(n, width)).astype(dtype)
    cols = np.sort(rng.choice(width, d_kept, replace=False))
    # n a power of two: weights, mean and centred values are dyadic, every product and partial sum exact
    fit = E.kde_fit(torch.from_numpy(x).to(dev), cols)
    want = np.atleast_2d(np.cov(x[:, cols].T.astype(np.float64), rowvar=1, bias=False, aweights=np.ones(n) / n))
    assert fit["rounds"] == 1
    assert np.array_equal(fit["covariance"].cpu().numpy(), want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 63, 64, 65, 300, 301])
@pytest.mark.parametrize("n", [1, 129, 60001])
def test_whitening_is_numpys_product_bit_for_bit(n, d, dtype):
    E, dev = _dev()
    rng = np.random.default_rng(n + d)
    width = d + 37
    x = rng.integers(-8, 9, size=(n, width)).astype(dtype)
    cols = rng.permutation(width)[:d].astype(np.int32)              # an unsorted column list
    mu = rng.integers(-3, 4, size=d).astype(np.float64)
    w = np.tril(rng.choice([0.0, 0.5, -0.5, 1.0, -2.0], size=(d, d)))
    w_dev = w.copy()
    w_dev[np.triu_indices(d, 1)] = np.nan                            # the upper triangle must never be read
    got = E.whiten_f64(torch.from_numpy(x).to(dev), torch.from_numpy(cols).to(dev), torch.from_numpy(mu).to(dev),
                       torch.from_numpy(w_dev).to(dev)).cpu().numpy()
    want = ((x[:, cols].astype(np.float64) - mu) @ w).astype(np.float32)    # exact: integers and halves < 2^24
    assert np.array_equal(got, want)


def _cond_data(n=6000, d=40, spread=1e4, seed=3):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(d, d)))
    return (rng.normal(size=(n, d)) * np.geomspace(1, spread, d)) @ q.T + 2.0


@pytest.mark.parametrize("case", ["relu_class", "cond_1e8"])
def test_fit_is_within_the_oracle_bounds(relu, case):
    E, dev = _dev()
    if case == "relu_class":
        x = np.ascontiguousarray(relu[:6000, 4:1604])
        cols = np.sort(np.argsort(np.var(x, axis=0))[-300:])
    else:
        x, cols = _cond_data(), None
    ref = K.fit(x, cols)
    assert not ref["prepare_failed"] and ref["rounds"] == 1
    fit = E.kde_fit(torch.from_numpy(x).to(dev), cols)
    assert fit["rounds"] == 1 and not fit["prepare_failed"]
    print(f"{case}: condition number of the covariance {K.kappa(ref['covariance']):.3g}")
    cov_b = K.cov_bound(x, cols)
    assert _report("covariance", np.abs(fit["covariance"].cpu().numpy() - ref["covariance"]), cov_b) <= 1
    w = fit["whitening"].cpu().numpy()
    w_b = K.whitening_bound(ref, cov_b)
    assert _report("whitening", np.linalg.norm(w - ref["whitening"]), w_b) <= 1
    res = ref["covariance"] * ref["factor"] ** 2 @ (w @ w.T) - np.eye(w.shape[0])
    assert _report("inverse residual", np.linalg.norm(res, 2), K.residual_bound(ref, cov_b)) <= 1
    assert _report("p", np.abs(fit["p"].cpu().numpy() - ref["p"]), K.p_bound(x, cols, ref, w_b)) <= 1
    assert abs(fit["log_det"] - ref["log_det"]) <= 1e-6 * max(1.0, abs(ref["log_det"]))


def test_golden_cases_with_the_device_fit(golden):
    from simple_tip_b200.core.surprise import LSA, MultiModalSA

    g = golden("lsa_reference.npz")
    for name, kw in (("plaus", {}), ("cube", {}), ("mf30", {"max_features": 30}), ("far", {})):
        sa = LSA(g[f"{name}.xtr"], backend="device", **kw)
        _close(sa(g[f"{name}.xte"]), g[f"{name}.lsa"])
        host = LSA(g[f"{name}.xtr"], **kw)
        assert np.array_equal(np.array(sa.removed_neurons), np.array(host.removed_neurons))
        assert sa.kde.prepare_failed == host.kde.prepare_failed is False
    assert np.array_equal(np.array(LSA(g["mf30.xtr"], max_features=30, backend="device").removed_neurons),
                          g["mf30.removed"])
    with pytest.warns(UserWarning, match="not able to fix"):
        sing = LSA(g["singular.xtr"], backend="device")
    assert sing.kde.prepare_failed and bool(g["singular.prepare_failed"])
    assert np.isinf(sing(g["singular.xte"])).all()
    mm = MultiModalSA.build_by_class(g["mf30.xtr"], g["pclsa.ytr"], lambda x, y: LSA(x, backend="device"))
    _close(mm(g["mf30.xte"], g["pclsa.pte"]), g["pclsa.lsa"])
    host = MultiModalSA.build_by_class(g["mf30.xtr"], g["pclsa.ytr"], lambda x, y: LSA(x))
    for mid, sa in mm.modal_sa.items():
        assert sa.removed_neurons == host.modal_sa[mid].removed_neurons
        assert sa.kde.prepare_failed == host.modal_sa[mid].kde.prepare_failed


def _outcome(x, backend, **kw):
    """(exception type and message or None, warning messages, prepare_failed, rounds) of one LSA fit"""
    from simple_tip_b200.core.surprise import LSA

    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        try:
            sa = LSA(x, backend=backend, **kw)
            err, failed = None, sa.kde.prepare_failed
        except Exception as e:            # noqa: BLE001 - the exception itself is the outcome compared
            err, failed = (type(e), str(e)), None
    msgs = [str(w.message) for w in rec if issubclass(w.category, UserWarning)]
    return err, msgs, failed


def _branch_case(kind):
    rng = np.random.default_rng(7)
    x = rng.normal(size=(400, 6))
    if kind == "one_row":
        return x[:1]
    if kind == "nan":
        x[3, 2] = np.nan
    elif kind == "inf":
        x[5, 1] = np.inf
    elif kind == "constant_column":
        x[:, 4] = 2.5
    elif kind == "duplicated_column":
        x[:, 5] = x[:, 0]
    elif kind == "n_le_d":
        x = x[:5]
    elif kind == "all_zero":
        x = np.zeros((50, 6))
    return x


@pytest.mark.parametrize("kind", ["one_row", "nan", "inf", "constant_column", "duplicated_column", "n_le_d",
                                  "all_zero", "max_features_half"])
def test_branch_cases_match_the_host_fit(kind):
    kw = {"max_features": 0.5} if kind == "max_features_half" else {}
    x = _branch_case(kind)
    host, dev = _outcome(x, "host", **kw), _outcome(x, "device", **kw)
    assert host == dev, (host, dev)
    expect = {"one_row": np.linalg.LinAlgError, "nan": np.linalg.LinAlgError, "inf": np.linalg.LinAlgError,
              "max_features_half": TypeError}
    if kind in expect:
        assert dev[0][0] is expect[kind]
        if dev[0][0] is np.linalg.LinAlgError:
            assert dev[0][1] == "Eigenvalues did not converge" and "Problem regarding KDE fitting" in dev[1]
    elif kind == "all_zero":
        assert dev[2] is False
    else:
        assert dev[2] is True and any("not able to fix" in m for m in dev[1])


def test_all_zero_matrix_fits_after_one_fill():
    E, dev = _dev()
    fit = E.kde_fit(torch.zeros((50, 6), dtype=torch.float64, device=dev))
    assert fit["rounds"] == 2 and not fit["prepare_failed"]


def test_cuda_traces_give_the_bits_of_numpy_traces():
    from simple_tip_b200.core.surprise import MultiModalSA

    E, dev = _dev()
    rng = np.random.default_rng(9)
    layers = [np.maximum(rng.normal(size=(3000, 4, 10)), 0).astype(np.float32),
              np.maximum(rng.normal(size=(3000, 30)), 0).astype(np.float32)]
    flat = np.concatenate([l.reshape(3000, -1) for l in layers], axis=1)
    probe = flat[:200] * 1.05
    y = rng.integers(0, 4, 3000)
    for backend in ("device", "host"):
        want = _lsa(flat, max_features=50, backend=backend)(probe)
        assert np.array_equal(_lsa(torch.from_numpy(flat).to(dev), max_features=50, backend=backend)(probe), want)
        cuda_layers = [torch.from_numpy(l).to(dev) for l in layers]
        assert np.array_equal(_lsa(cuda_layers, max_features=50, backend=backend)(probe), want)
    want = _lsa(flat, max_features=50, backend="device")(probe)
    assert np.array_equal(_lsa(flat, max_features=50, backend="device")(probe), want)        # repeated fits
    ctor = lambda x, _: _lsa(x, max_features=50, backend="device")                        # noqa: E731
    pc_np = MultiModalSA.build_by_class(flat, y, ctor)
    pc_dev = MultiModalSA.build_by_class(torch.from_numpy(flat).to(dev), torch.from_numpy(y).to(dev), ctor)
    assert all(isinstance(sa.kde.__dict__.get("_lazy"), dict) for sa in pc_dev.modal_sa.values())
    py = y[:200]
    assert np.array_equal(pc_dev(probe, py), pc_np(probe, py))


def test_forward_hook_traces_fit_lsa_without_leaving_hbm():
    _, dev = _dev()
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(20, 64), torch.nn.ReLU(), torch.nn.Linear(64, 32), torch.nn.ReLU()).to(dev)
    seen = []
    model[1].register_forward_hook(lambda m, i, o: seen.append(o.detach()))
    model[3].register_forward_hook(lambda m, i, o: seen.append(o.detach()))
    with torch.no_grad():
        model(torch.randn(4000, 20, device=dev))
    sa = _lsa(seen, max_features=40, backend="device")
    assert "dataset" in sa.kde.__dict__["_lazy"]              # the training rows were never copied to the host
    assert sa.kde._engine.n == 4000
    flat = torch.cat(seen, dim=1).cpu().numpy()
    probe = flat[:100]
    assert np.array_equal(sa(probe), _lsa(flat, max_features=40, backend="device")(probe))
    host = _lsa(flat, max_features=40)
    assert sa.removed_neurons == host.removed_neurons
    np.testing.assert_allclose(sa.kde.dataset, host.kde.dataset, rtol=0, atol=0)
    _close(sa(probe), host(probe))
