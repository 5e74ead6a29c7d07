"""GPU: the device EmpiricalCovariance fit (csrc/covariance.cu, engine.cov_*, core/covariance.py) against NumPy,
scipy, sklearn and the float64 restatement of oracle/cov_oracle.py.  Bounds come from DESIGN.md §5c; every bounded
comparison prints the measured error as a fraction of its bound."""
import os
import warnings

import numpy as np
import pytest
from scipy import linalg

from oracle import cov_oracle as C

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TWO53 = 2.0 ** 53


def _dev():
    from simple_tip_b200 import engine as E

    return E, E.require_cuda()


def _fit(x):
    from simple_tip_b200.core.covariance import EmpiricalCovariance

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return EmpiricalCovariance().fit(x)


def _report(name, err, bound):
    frac = float(np.max(err / bound, initial=0.0))
    print(f"{name}: worst error = {frac:.3g} of the bound")
    return frac


@pytest.fixture(scope="module")
def big():
    rng = np.random.default_rng(11)
    return rng.normal(size=(60000, 2304)) * rng.uniform(0.1, 30, size=2304) + rng.normal(size=2304) * 5


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 17, 1600, 2304])
@pytest.mark.parametrize("n", [1, 2, 6000, 60000])
def test_location_is_numpys_mean_bit_for_bit(big, n, d, dtype):
    E, dev = _dev()
    x = np.ascontiguousarray(big[:n, :d]).astype(dtype)
    loc, mean, flags = E.cov_location(torch.from_numpy(x).to(dev))
    assert loc.dtype == torch.from_numpy(x).dtype and np.array_equal(loc.cpu().numpy(), x.mean(0))
    assert np.array_equal(mean.cpu().numpy(), np.array(x.T, ndmin=2, dtype=np.float64).mean(axis=1))
    assert int(flags.item()) == 0


def test_non_finite_input_raises_sklearns_error():
    x = np.random.default_rng(1).normal(size=(100, 5)).astype(np.float32)
    x[7, 3] = np.nan
    with pytest.raises(ValueError, match="Input X contains NaN"):
        _fit(x)
    x[7, 3] = np.inf
    with pytest.raises(ValueError, match=r"Input X contains infinity or a value too large for dtype\('float32'\)"):
        _fit(x)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,d", [(2, 1), (1024, 17), (4096, 300), (16384, 1600)])
def test_covariance_is_np_cov_bit_for_bit_on_exact_data(n, d, dtype):
    x = np.random.default_rng(n + d).integers(-8, 9, size=(n, d)).astype(dtype)
    # n a power of two: the mean is dyadic; |n (x - m)| <= 16 n, so every scaled product is below 256 n^2 and every
    # partial sum below 256 n^3 < 2^53: each order of summation is exact
    assert n & (n - 1) == 0 and 256.0 * n ** 3 < TWO53
    ec = _fit(x)
    assert np.array_equal(ec.covariance_, np.cov(x.T, bias=1).reshape(d, d))
    assert np.array_equal(ec.location_, x.mean(0))


def _relu_rows(n, d, seed, dtype=np.float32):
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.normal(size=(n, d)) + rng.normal(size=d), 0.0)
    x[:, : max(1, d // 32)] = 0.0
    return x.astype(dtype)


@pytest.mark.parametrize("n,d,dtype,kind", [(6000, 128, np.float32, "relu"), (6000, 1600, np.float32, "relu"),
                                            (2000, 64, np.float64, "normal"), (6000, 300, np.float32, "normal")])
def test_covariance_precision_and_scores_within_the_oracle_bounds(n, d, dtype, kind):
    if kind == "relu":
        x = _relu_rows(n, d, seed=d)
    else:
        rng = np.random.default_rng(d)
        x = (rng.normal(size=(n, d)) * rng.uniform(0.5, 3, size=d) + rng.normal(size=d)).astype(dtype)
    ec = _fit(x)
    ref = C.fit(x)
    cov_b = C.scatter_bound(x, ref["covariance"])
    _report(f"{kind} {n}x{d} covariance", np.abs(ec.covariance_ - ref["covariance"]), cov_b + 1e-300)
    assert np.all(np.abs(ec.covariance_ - ref["covariance"]) <= cov_b)
    assert np.array_equal(ec._dev["live"].cpu().numpy(), ref["live"])
    s = linalg.eigvalsh(np.cov(x.T, bias=1))
    if C.gap(s, C.cutoff(s, d)) > C.RANK_GAP:
        assert ec.rank_ == ref["rank"] == int(np.sum(np.abs(s) > C.cutoff(s, d)))
    assert ec.rank_ == ref["rank"]
    pb = C.precision_bound(x, ref, cov_b)
    _report("  precision", np.abs(ec.precision_ - ref["precision"]), np.full(1, pb))
    assert np.max(np.abs(ec.precision_ - ref["precision"])) <= pb
    test = x[: min(n, 1000)] * 1.1
    sb = C.score_bound(test, ref, pb)
    err = np.abs(ec.mahalanobis(test) - C.scores(test, ref))
    _report("  scores", err, sb + 1e-300)
    assert np.all(err <= sb)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("kind", C.RANK_CASES)
def test_rank_equals_scipys(kind, dtype):
    x = C.rank_case(kind, seed=1, dtype=dtype)
    d = x.shape[1]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cov = np.cov(x.T, bias=1).reshape(d, d)
    p, rank = linalg.pinvh(cov, return_rank=True)
    s = linalg.eigvalsh(cov)
    assert C.gap(s, C.cutoff(s, d)) > C.RANK_GAP
    ec = _fit(x)
    assert ec.rank_ == rank
    if kind in ("one_row", "constant"):
        assert not ec.covariance_.any() and not ec.precision_.any()
        assert not np.any(ec.mahalanobis(x[:5] + 1.0))


def test_one_row_warns_as_sklearn_does():
    from simple_tip_b200.core.covariance import EmpiricalCovariance

    with pytest.warns(UserWarning, match="Only one sample available"):
        ec = EmpiricalCovariance().fit(np.ones((1, 3), np.float32))
    assert ec.location_.dtype == np.float32 and not ec.precision_.any()


def test_mdsa_device_meets_the_golden_and_live_sklearn(golden):
    from simple_tip_b200.core.surprise import MDSA, MultiModalSA

    g = golden("mdsa_mlsa_reference.npz")
    xtr, ytr, xte, pte = g["x.xtr"], g["x.ytr"], g["x.xte"], g["x.pte"]
    m = MDSA(xtr, backend="device")
    np.testing.assert_allclose(m(xte), g["mdsa.out"], rtol=1e-4)
    from sklearn.covariance import EmpiricalCovariance

    sk = EmpiricalCovariance().fit(xtr)
    np.testing.assert_allclose(m(xte), sk.mahalanobis(xte), rtol=1e-4)
    assert np.array_equal(m.covariance_matrix.location_, sk.location_)
    pc = MultiModalSA.build_by_class(xtr, ytr, lambda x, y: MDSA(x, backend="device"))
    np.testing.assert_allclose(pc(xte, pte), g["pcmdsa.out"], rtol=1e-4)
    out32 = MDSA(xtr.astype(np.float32), backend="device")(xte.astype(np.float32))
    assert out32.dtype == np.float64
    np.testing.assert_allclose(out32, g["mdsa.out"], rtol=2e-4)
    sing = MDSA(g["sing.xtr"], backend="device")
    np.testing.assert_allclose(sing(g["sing.xte"]), g["sing.out"], rtol=1e-4, atol=1e-6)
    cov = EmpiricalCovariance().fit(g["sing.xtr"]).covariance_
    s = linalg.eigvalsh(cov)
    if C.gap(s, C.cutoff(s, cov.shape[0])) > C.RANK_GAP:
        assert sing.covariance_matrix.rank_ == linalg.pinvh(cov, return_rank=True)[1]
    with pytest.raises(ValueError):
        m(xte[:, :5])


def test_pc_mdsa_and_pc_mmdsa_conformance_through_the_environment_variable(monkeypatch):
    """The MDSA rows of test_reference_conformance.py, re-run with B200TIP_COV=device."""
    from simple_tip_b200.core.surprise import MDSA, MultiModalSA

    monkeypatch.setenv("B200TIP_COV", "device")
    rng = np.random.RandomState(42)
    acts = rng.random((100, 10))
    sa = MDSA(acts)
    assert sa.backend == "device"
    id_sa, ood_sa = sa(acts[:10]), sa(acts[:10] + 10)
    assert np.all(ood_sa > id_sa) and np.all(id_sa >= 0) and id_sa.shape == (10,)
    big = np.concatenate([acts for _ in range(100)])
    first = sa(big).reshape((100, -1))
    assert np.all(first == first[0]) and np.all(sa(big).reshape((100, -1)) == first)
    rng = np.random.RandomState(42)
    acts = rng.random((20000, 10))
    np.testing.assert_allclose(MDSA(acts).covariance_matrix.covariance_, np.cov(acts.T), 0.1)
    for _ in range(3):
        rng.random((2000, 10))
    two = np.concatenate([rng.random((100, 10)), rng.random((100, 10)) + 0.9])
    pts = np.array([[0.5] * 10, [1.4] * 10])
    monkeypatch.setenv("B200TIP_KMEANS", "device")
    mm = MultiModalSA.build_with_kmeans(two, None, lambda x, _: MDSA(x), potential_k=[2, 3, 4])
    assert all(m.backend == "device" for m in mm.modal_sa.values())
    assert np.all(mm(pts + 2, None) > mm(pts, None))
    labels = rng.randint(0, 3, size=600)
    x = rng.random((600, 10)) + labels[:, None]
    pc = MultiModalSA.build_by_class(x, labels, lambda a, y: MDSA(a))
    for c, m in pc.modal_sa.items():
        assert m.backend == "device"
        np.testing.assert_allclose(pc(x, labels)[labels == c], m(x[labels == c]), rtol=0)


def test_cuda_tensor_input_gives_the_same_bits_and_two_fits_agree():
    E, dev = _dev()
    x = _relu_rows(6000, 300, seed=5)
    a, b = _fit(x), _fit(x)
    t = _fit(torch.from_numpy(x).to(dev))
    for other in (b, t):
        for name in ("location_", "covariance_", "precision_"):
            assert np.array_equal(getattr(a, name), getattr(other, name)), name
        assert a.rank_ == other.rank_
    test = x[:500] + 0.25
    assert np.array_equal(a.mahalanobis(test), t.mahalanobis(torch.from_numpy(test).to(dev)).cpu().numpy())
    assert np.array_equal(a.mahalanobis(test), b.mahalanobis(test))
