"""The surprise-adequacy arm on the GPU: the one-pass SC-CAM kernel (`cam_from_surprise`), the multimodal SAs on
CUDA traces, and `SurpriseHandler.evaluate_all` through the result files."""
import numpy as np
import pytest

from oracle import np_oracle, sc_oracle
from tests.test_sc_cam_oracle import CASES

pytestmark = pytest.mark.gpu


def _torch():
    import torch

    return torch


def _dense_cam(values, mapper):
    from simple_tip_b200.core.prioritizers import cam

    return np.array(list(cam(values, mapper.get_coverage_profile(values))), dtype=np.int64)


def _sc_cam(values, mapper):
    from simple_tip_b200.core.prioritizers import cam_from_surprise

    return np.array(list(cam_from_surprise(values, mapper)), dtype=np.int64)


def _both_inputs(values):
    torch = _torch()
    return [values, torch.from_numpy(values).cuda()]


# ------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,values,sections,overflow", CASES, ids=[c[0] for c in CASES])
def test_sc_cam_equals_dense_cam_and_oracle(name, values, sections, overflow):
    from simple_tip_b200.core import prioritizers as P
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    ub = np.max(values) if not np.isnan(values).any() else 2.5
    mapper = SurpriseCoverageMapper(sections, ub, overflow)
    want = np_oracle.cam_oracle(values, mapper.get_coverage_profile(values))
    assert np.array_equal(_dense_cam(values, mapper), want)
    assert np.array_equal(sc_oracle.sc_cam_oracle(values, mapper.thresholds), want)
    for v in _both_inputs(values):
        assert np.array_equal(_sc_cam(v, mapper), want), type(v)
        assert P.LAST_GREEDY_PICKS == np.unique(sc_oracle.sc_buckets(values, mapper.thresholds)[
            sc_oracle.sc_buckets(values, mapper.thresholds) >= 0]).size


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [0, 1, 10_000])
def test_sc_cam_sizes(dtype, n):
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    rng = np.random.default_rng(n)
    values = (rng.gamma(2.0, size=n) * 3).astype(dtype)
    if n >= 10:
        values[rng.integers(0, n, n // 10)] = values[:n // 10]          # repeated values
    for overflow in (False, True):
        mapper = SurpriseCoverageMapper(1000, np.max(values) if n else 1.0, overflow)
        # (the dense profile of no sample cannot be flattened: the reference's cam fails there)
        want = np_oracle.cam_oracle(values, mapper.get_coverage_profile(values)) if n else np.zeros(0, np.int64)
        for v in _both_inputs(values):
            assert np.array_equal(_sc_cam(v, mapper), want)


def test_sc_cam_golden(golden):
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    s = golden("siblings_reference.npz")
    v = s["sc.values"]
    for x in _both_inputs(v):
        assert np.array_equal(_sc_cam(x, SurpriseCoverageMapper(1000, np.max(v))), s["sc.cam"])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_sc_cam_one_million_against_the_closed_form(dtype):
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    rng = np.random.default_rng(7)
    values = np.round(rng.gamma(2.0, size=1_000_000) * 50, 2).astype(dtype)           # many repeated values
    values[rng.integers(0, values.size, 1000)] = np.nan
    for overflow in (False, True):
        mapper = SurpriseCoverageMapper(1000, np.nanmax(values) * 0.9, overflow)
        want = sc_oracle.sc_cam_oracle(values, mapper.thresholds)
        for v in _both_inputs(values):
            assert np.array_equal(_sc_cam(v, mapper), want)


def _failing_cases():
    """A DSA score vector holding NaN (test rows of a class the training set lacks) and an LSA score vector holding
    +inf (the KDE density underflows far from the training rows)."""
    from simple_tip_b200.core.surprise import DSA, LSA

    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(1500, 300, 16, 4, seed=3)
    pte = pte.copy()
    pte[::17] = 4
    dsa = DSA(xtr, ytr)(xte, pte)
    lsa = LSA(xtr)(np.concatenate([xte, xte[:20] + 1e3]))
    assert np.isnan(dsa).any() and np.isinf(lsa).any()
    return {"dsa": dsa, "lsa": lsa}


@pytest.mark.parametrize("overflow", [False, True])
def test_sc_cam_non_monotone_thresholds_take_the_dense_path(overflow):
    from simple_tip_b200.core.prioritizers import thresholds_one_hot
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    rng = np.random.default_rng(1)
    generic = rng.normal(size=500).astype(np.float32) * 3
    generic[::50] = np.nan
    vectors = dict(_failing_cases(), generic=generic)
    with np.errstate(invalid="ignore"):
        for name, v in vectors.items():
            for ub in (0.0, -1.0, np.nan, np.inf, np.max(v)):
                mapper = SurpriseCoverageMapper(1000, ub, overflow)
                if ub != 0.0:
                    assert not thresholds_one_hot(mapper.thresholds), (name, ub)
                want = np_oracle.cam_oracle(v, mapper.get_coverage_profile(v))
                for x in _both_inputs(v):
                    assert np.array_equal(_sc_cam(x, mapper), want), (name, ub, overflow)


def test_sc_cam_rejects_too_many_sections_before_any_launch():
    from simple_tip_b200 import _lib
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper

    v = np.linspace(0, 1, 100)
    assert np.array_equal(_sc_cam(v, SurpriseCoverageMapper(_lib.SC_CAM_MAX_SECTIONS, 1.0)),
                          np_oracle.cam_oracle(v, SurpriseCoverageMapper(_lib.SC_CAM_MAX_SECTIONS, 1.0)
                                               .get_coverage_profile(v)))
    before = _lib.launch_count()
    for x in _both_inputs(v):
        with pytest.raises(ValueError):
            _sc_cam(x, SurpriseCoverageMapper(_lib.SC_CAM_MAX_SECTIONS + 1, 1.0))
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------
# multimodal SAs on CUDA traces
# ------------------------------------------------------------------------------------------
def _seeded(fn, seed):
    np.random.seed(seed)          # sklearn's unseeded KMeans / GaussianMixture draw from NumPy's global RNG
    return fn()


@pytest.mark.parametrize("kind", ["lsa", "mdsa", "mlsa", "kmeans"])
def test_multimodal_sa_takes_cuda_traces(kind):
    torch = _torch()
    from simple_tip_b200.core.surprise import LSA, MDSA, MLSA, MultiModalSA

    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(1500, 300, 16, 4, seed=5)
    ctor = {"lsa": lambda x, y: LSA(x), "mdsa": lambda x, y: MDSA(x),
            "mlsa": lambda x, y: MLSA(x, num_components=3), "kmeans": lambda x, y: MDSA(x)}[kind]

    def build(x):
        if kind == "kmeans":
            return MultiModalSA.build_with_kmeans(x, ytr, ctor, potential_k=range(2, 5), subsampling=0.3,
                                                  backend="sklearn")
        return MultiModalSA.build_by_class(x, ytr, ctor)

    host = _seeded(lambda: build(xtr), 11)
    want = _seeded(lambda: host(xte, pte), 12)
    # a list of hook layers (two column blocks) and one tensor
    dev_layers = [torch.from_numpy(np.ascontiguousarray(xtr[:, :6])).cuda(),
                  torch.from_numpy(np.ascontiguousarray(xtr[:, 6:])).cuda()]
    dev = _seeded(lambda: build(dev_layers), 11)
    if kind == "kmeans":
        assert dev.discriminator.best_k == host.discriminator.best_k
    got = _seeded(lambda: dev(torch.from_numpy(xte).cuda(), torch.from_numpy(pte).cuda()), 12)
    np.testing.assert_array_equal(got, want)
    te_layers = [torch.from_numpy(np.ascontiguousarray(xte[:, :6])).cuda(),
                 torch.from_numpy(np.ascontiguousarray(xte[:, 6:])).cuda()]
    np.testing.assert_array_equal(_seeded(lambda: dev(te_layers, pte), 12), want)


# ------------------------------------------------------------------------------------------
# the handler
# ------------------------------------------------------------------------------------------
def _toy_model(torch):
    """A small conv net whose last bias is shifted so that it predicts its 6 classes about equally often on normal
    noise (random weights alone predict one class for almost every input)."""
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Conv2d(1, 4, 3), torch.nn.ReLU(), torch.nn.MaxPool2d(2), torch.nn.Flatten(),
                                torch.nn.Linear(4 * 5 * 5, 24), torch.nn.ReLU(), torch.nn.Linear(24, 6),
                                torch.nn.Softmax(dim=1)).cuda().eval()
    x = torch.from_numpy(np.random.default_rng(99).normal(size=(20_000, 1, 12, 12)).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x).double().cpu().numpy()
    bias, step = np.zeros(6), z.std(axis=0).mean()
    for it in range(500):
        freq = np.bincount((z + bias).argmax(axis=1), minlength=6) / z.shape[0]
        bias -= step * 2.0 * (freq - 1 / 6) * 0.99 ** it
    with torch.no_grad():
        model[-2].bias += torch.from_numpy(bias).float().cuda()
    return model


def _balanced_inputs(torch, model, per_class, rng, scale=1.0, pool=40_000):
    """`per_class` inputs of every class the model predicts often enough, each with a clear top-1 margin of the
    pre-softmax outputs so that batching cannot flip the prediction."""
    x = torch.from_numpy((rng.normal(size=(pool, 1, 12, 12)) * scale).astype(np.float32)).cuda()
    with torch.no_grad():
        z = model[:-1](x)
    top = z.topk(2, dim=1).values
    pred = z.argmax(dim=1).cpu().numpy()
    clear = ((top[:, 0] - top[:, 1]) > 1e-3).cpu().numpy()
    rows = {c: np.flatnonzero((pred == c) & clear)[:per_class] for c in range(z.shape[1])}
    return {c: x[torch.from_numpy(r).cuda()] for c, r in rows.items() if r.size == per_class}


def _handler_run(monkeypatch, kmeans_backend):
    torch = _torch()
    from simple_tip_b200.core.surprise_handler import SurpriseHandler

    if kmeans_backend is not None:
        monkeypatch.setenv("B200TIP_KMEANS", kmeans_backend)
    model = _toy_model(torch)
    rng = np.random.default_rng(0)
    pools = [_balanced_inputs(torch, model, 150 + 2 * 40, rng), _balanced_inputs(torch, model, 40, rng, scale=1.3)]
    classes = sorted(set(pools[0]) & set(pools[1]))
    assert len(classes) >= 3, "the toy model predicts too few classes"
    xtr = torch.cat([pools[0][c][:150] for c in classes])
    datasets = {"nominal": torch.cat([pools[0][c][150:190] for c in classes]),
                "ood": torch.cat([pools[1][c] for c in classes])}
    h = SurpriseHandler(model, [4], xtr, batch_size=64)
    h.fitted = {}
    h.TESTED_SA = {name: (lambda x, y, name=name, fit=fit: h.fitted.setdefault(name, fit(x, y)))
                   for name, fit in SurpriseHandler.TESTED_SA.items()}
    seen = {}
    collect = h._acti_and_pred

    def spy(data):
        ats, pred = collect(data)
        seen[id(data)] = (ats, pred)
        return ats, pred
    h._acti_and_pred = spy
    np.random.seed(2024)
    res = h.evaluate_all(datasets, dsa_badge_size=7)
    test = {name: seen[id(x)] for name, x in datasets.items()}
    return h, res, test


def _host_reference(h, test):
    """The same TESTED_SA entries on host copies of the same traces, drawing the same global-RNG numbers."""
    train_ats = [a.cpu().numpy() for a in h.train_ats]
    np.random.seed(2024)
    out = {}
    for sa_name, sa_func in type(h).TESTED_SA.items():
        sa = sa_func(train_ats, h.train_pred)
        out[sa_name] = {ds: sa([a.cpu().numpy() for a in ats], pred) for ds, (ats, pred) in test.items()}
    return out


@pytest.mark.parametrize("kmeans_backend", [None, "device"])
def test_surprise_handler(monkeypatch, kmeans_backend):
    from simple_tip_b200.core.surprise import DSA, SurpriseCoverageMapper
    from simple_tip_b200.core.surprise_handler import NUM_SC_BUCKETS

    h, res, test = _handler_run(monkeypatch, kmeans_backend)
    assert all(a.is_cuda for a in h.train_ats) and h.train_pred.dtype == np.int64
    assert list(res) == ["dsa", "pc-lsa", "pc-mdsa", "pc-mlsa", "pc-mmdsa"]
    ref = _host_reference(h, test)
    for sa_name, per_ds in res.items():
        assert list(per_ds) == ["nominal", "ood"]
        for ds, (scores, order, times) in per_ds.items():
            assert isinstance(scores, np.ndarray) and scores.shape == (test[ds][1].shape[0],)
            want = ref[sa_name][ds]
            assert scores.dtype == want.dtype
            if sa_name == "dsa":
                np.testing.assert_array_equal(scores, want)
            else:
                np.testing.assert_allclose(scores, want, rtol=1e-4, atol=1e-6)
            mapper = SurpriseCoverageMapper(NUM_SC_BUCKETS, np.max(scores))
            assert np.array_equal(order, np_oracle.cam_oracle(scores, mapper.get_coverage_profile(scores)))
            assert len(times) == 4 and all(t >= 0 for t in times), times
    assert isinstance(h.fitted["dsa"], DSA) and h.fitted["dsa"].badge_size == 7


def test_surprise_arm_result_files(monkeypatch, tmp_path):
    from simple_tip_b200.core import results as R
    from simple_tip_b200.core.apfd import apfd_from_order
    from simple_tip_b200.core.surprise import SurpriseCoverageMapper
    from simple_tip_b200.core.surprise_handler import NUM_SC_BUCKETS

    _, res, test = _handler_run(monkeypatch, None)
    out = str(tmp_path)
    rng = np.random.default_rng(5)
    mis = {ds: rng.random(pred.shape[0]) < 0.3 for ds, (_, pred) in test.items()}
    for ds, m in mis.items():
        R.persist(out, "toy", ds, "is_misclassified", 0, m)
    for sa_name, per_ds in res.items():
        for ds, (scores, order, times) in per_ds.items():
            R.persist_tip(out, "toy", ds, 0, sa_name, scores, order, times)
    for ds, m in mis.items():
        apfd = R.load_apfd_values(out, "toy", ds)
        for sa_name, per_ds in res.items():
            scores = per_ds[ds][0]
            prof = SurpriseCoverageMapper(NUM_SC_BUCKETS, np.max(scores)).get_coverage_profile(scores)
            assert apfd[sa_name][0] == apfd_from_order(m, np.argsort(-scores))
            assert apfd[sa_name + "-cam"][0] == apfd_from_order(m, np_oracle.cam_oracle(scores, prof))
            assert R.load_times(out, "toy", ds, 0, sa_name) == per_ds[ds][2]
