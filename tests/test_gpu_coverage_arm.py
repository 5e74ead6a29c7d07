"""The neuron-coverage arm on the GPU: `KMNC.packed` (libb200tip `tip_kmnc_packed`) on every kernel route against the
dense profile and the bucket ids, KMNC's CAM from the packed bits, and `CoverageWorker.evaluate_all` against the
metrics on host copies of the same traces, through the result files."""
import copy

import numpy as np
import pytest

from oracle import coverage_oracle as CO
from oracle import np_oracle

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64


def _torch():
    import torch

    return torch


# ------------------------------------------------------------------------------------------
# KMNC.packed
# ------------------------------------------------------------------------------------------
def _kmnc_case(n, d, sections, adt, sdt, seed):
    """ReLU-like activations against statistics with min = 0 (so a == min is common), negative minima, constant
    neurons (jump 0), values exactly on every threshold, and NaN rows."""
    rng = np.random.default_rng(seed)
    mins = np.zeros(d, dtype=sdt)
    mins[rng.random(d) < 0.2] = -rng.random() - 0.5
    maxs = (mins + rng.random(d) * 3 + 0.1).astype(sdt)
    const = rng.random(d) < 0.05
    maxs[const] = mins[const]
    act = np.maximum(rng.normal(size=(n, d)) * 1.5, mins - 0.25).astype(adt)
    if n:
        jumps = (maxs - mins) / sections
        thresh = [(mins + jumps * 0) + jumps * i for i in range(sections + 1)]
        pick = rng.random((n, d)) < 0.15
        which = rng.integers(0, sections + 1, size=(n, d))
        on_edge = np.choose(which, thresh).astype(adt)
        act[pick] = on_edge[pick]
        act[rng.random((n, d)) < 0.1] = 0                    # ReLU zeros: a == min for most neurons
        act[rng.integers(0, n, size=max(1, n // 50))] = np.nan
    return act, mins, maxs


# (name, n, d, activation dtype, statistics dtype, element offset of a CUDA view)
ROUTES = [
    ("strip", 4096, 2052, f32, f32, 0),          # column-strip kernel, several strips, d % 128 != 0
    ("strip_partial_warp", 64, 300, f32, f32, 0),
    ("vec4", 17, 300, f32, f32, 0),
    ("vec4_one_row", 1, 2052, f32, f32, 0),
    ("generic_d", 40, 301, f32, f32, 0),         # d % 4 != 0
    ("generic_view", 40, 300, f32, f32, 1),      # 4-byte aligned view of a CUDA allocation
    ("f64_activations", 40, 300, f64, f32, 0),
    ("f64_statistics", 40, 300, f32, f64, 0),
    ("f64_both", 33, 129, f64, f64, 0),
    ("empty", 0, 300, f32, f32, 0),
]


def _inputs(act, off):
    """the activations as the tests hand them over: NumPy (unless a view is asked for) and a CUDA tensor"""
    torch = _torch()
    n, d = act.shape
    flat = np.concatenate([np.zeros(off, act.dtype), act.ravel(), np.zeros(4, act.dtype)])
    view = torch.from_numpy(flat).cuda()[off:off + n * d].view(n, d)
    return ([] if off else [act]) + [view]


def _pack_planes(profile):
    """dense [n, d, planes] -> tip_kmnc_packed's words: pack_cover's single-plane layout, plane after plane"""
    return np.concatenate([CO.pack_cover(profile[..., s]) for s in range(profile.shape[2])], axis=1)


def _one_hot(bucket, sections):
    n, d = bucket.shape
    prof = np.zeros((n, d, sections), dtype=bool)
    np.put_along_axis(prof, np.maximum(bucket, 0).astype(np.int64)[..., None], (bucket >= 0)[..., None], axis=2)
    return prof


@pytest.mark.parametrize("sections", [1, 2, 3, 7])
@pytest.mark.parametrize("name,n,d,adt,sdt,off", ROUTES, ids=[r[0] for r in ROUTES])
def test_kmnc_packed_equals_buckets_and_dense_profile(name, n, d, adt, sdt, off, sections):
    from simple_tip_b200.core.neuron_coverage import KMNC

    act, mins, maxs = _kmnc_case(n, d, sections, adt, sdt, seed=d + sections)
    kmnc = KMNC([mins], [maxs], sections)
    if n:
        with np.errstate(invalid="ignore"):
            want_score, want_prof = np_oracle.kmnc_oracle([mins], [maxs], sections, act)
    else:           # (the oracle's sum over a reshaped empty profile is undefined)
        want_score, want_prof = np.zeros(0, np.int32), np.zeros((0, d, sections), bool)
    for x in _inputs(act, off):
        score, bits = kmnc.packed(x)
        assert score.is_cuda and bits.is_cuda and score.dtype == bits.dtype == _torch().int32
        assert tuple(bits.shape) == (n, sections * CO.packed_words(d)) and tuple(score.shape) == (n,)
        b = bits.cpu().numpy().view(np.uint32)
        got = CO.unpack_cover(b, d, planes=sections)
        got = got if sections > 1 else got[..., None]
        assert np.array_equal(got, want_prof), (name, type(x))
        assert np.array_equal(_pack_planes(want_prof), b), (name, "padding bits")
        assert np.array_equal(score.cpu().numpy(), want_score.astype(np.int32)), name
        if n:
            b_score, bucket = kmnc.buckets(x)
            assert np.array_equal(_one_hot(bucket, sections), got) and np.array_equal(b_score, want_score)
            d_score, d_prof = kmnc(x)
            assert np.array_equal(d_prof, got) and np.array_equal(d_score, want_score)


@pytest.mark.parametrize("sections", [2, 7])
def test_kmnc_cam_from_packed_bits(sections):
    from simple_tip_b200.core.neuron_coverage import KMNC
    from simple_tip_b200.core.prioritizers import cam_from_bits, cam_from_buckets

    act, mins, maxs = _kmnc_case(3000, 520, sections, f32, f32, seed=11)
    act = np.nan_to_num(act)
    kmnc = KMNC([mins], [maxs], sections)
    scores, prof = kmnc(act)
    want = np_oracle.cam_oracle(scores, prof)
    _, bits = kmnc.packed(act)
    assert np.array_equal(np.array(list(cam_from_bits(scores, bits)), dtype=np.int64), want)
    _, bucket = kmnc.buckets(act, device_out=True)
    assert np.array_equal(np.array(list(cam_from_buckets(scores, bucket, sections)), dtype=np.int64), want)


def test_kmnc_packed_rejects_rows_beyond_cam_from_bits_before_any_launch():
    from simple_tip_b200 import _lib
    from simple_tip_b200.core.neuron_coverage import KMNC

    mins, maxs = np.zeros(4, f32), np.ones(4, f32)
    act = np.full((3, 4), 0.5, f32)
    before = _lib.launch_count()
    for x in (act, _torch().from_numpy(act).cuda()):
        with pytest.raises(ValueError):
            KMNC([mins], [maxs], 2 ** 29).packed(x)           # 2^29 sections x 4 words = 2^31 words per row
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------
# the worker
# ------------------------------------------------------------------------------------------
NAMES = ["NBC_0", "NBC_0.5", "NBC_1", "SNAC_0", "SNAC_0.5", "SNAC_1", "NAC_0", "NAC_0.75", "TKNC_1", "TKNC_2",
         "TKNC_3", "KMNC_2"]
NC_LAYERS = [1, 2]          # the toy net's ReLU and max-pool: 400 + 100 neurons
BATCH = 64


def _toy_model(torch):
    from tests.test_gpu_surprise_arm import _toy_model as toy

    return toy(torch)


def _data():
    rng = np.random.default_rng(42)
    train = rng.normal(size=(1500, 1, 12, 12)).astype(f32)
    sets = {"nominal": rng.normal(size=(700, 1, 12, 12)).astype(f32),
            "ood": (rng.normal(size=(450, 1, 12, 12)) * 1.3 + 0.2).astype(f32)}
    return train, sets


def _run(model, train, sets, as_numpy):
    """worker + evaluate_all per set; also the test traces the worker scored (spied), as host arrays"""
    torch = _torch()
    from simple_tip_b200.core.coverage_worker import CoverageWorker

    def to_input(x):
        return x if as_numpy else torch.from_numpy(x).cuda()
    w = CoverageWorker(model, NC_LAYERS, to_input(train), batch_size=BATCH)
    seen = []
    traces = w._traces

    def spy(data):
        layers, flat = traces(data)
        seen.append((layers, flat))
        return layers, flat
    w._traces = spy
    res, host = {}, {}
    for ds, x in sets.items():
        res[ds] = w.evaluate_all(to_input(x), ds)
        layers, flat = seen[-1]
        assert all(a.is_cuda for a in layers) and flat.is_cuda
        host[ds] = [a.cpu().numpy() for a in layers]
        assert np.array_equal(flat.cpu().numpy(), np_oracle.flatten_rows(host[ds]))
    return w, res, host


def _host_train_traces(model, train):
    """the training badges' hooked layers as host arrays, badge by badge as the worker walks them"""
    torch = _torch()
    from simple_tip_b200.core.activations import TransparentModel

    tm = TransparentModel(model, NC_LAYERS, include_last_layer=False)
    dev = next(model.parameters()).device
    return [[a.cpu().numpy() for a in tm.get_activations(torch.from_numpy(train[s:s + BATCH]).to(dev))]
            for s in range(0, train.shape[0], BATCH)]


def _check(w, res, host, badges):
    from simple_tip_b200.core.aggregate_statistics import AggregateStatisticsCollector

    # statistics: bit for bit those of the host restatement and of the collector fed the host badges
    col = AggregateStatisticsCollector()
    for b in badges:
        col.track(b)
    o_min, o_max, o_std = np_oracle.stats_oracle(badges)
    c_min, c_max, c_std = col.get()
    for got, want, want_c in zip(w.mins + w.maxs + w.stds, o_min + o_max + o_std, c_min + c_max + c_std):
        assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want, equal_nan=True)
        assert np.array_equal(got, want_c, equal_nan=True)
    assert list(w.metrics) == NAMES
    for ds, (times, scores, orders) in res.items():
        assert list(times) == list(scores) == list(orders) == NAMES
        for name, metric in w.metrics.items():
            want_s, want_p = metric(host[ds])
            assert isinstance(scores[name], np.ndarray) and scores[name].dtype == want_s.dtype, (ds, name)
            assert np.array_equal(scores[name], want_s), (ds, name)
            assert orders[name].dtype == np.int64
            assert np.array_equal(orders[name], np_oracle.cam_oracle(want_s, want_p)), (ds, name)
            assert len(times[name]) == 4 and all(t >= 0 for t in times[name]), (ds, name, times[name])


@pytest.fixture(scope="module")
def worker_run():
    torch = _torch()
    model = _toy_model(torch)
    train, sets = _data()
    return model, train, sets, _run(model, train, sets, as_numpy=False)


def test_coverage_worker_on_cuda_inputs(worker_run):
    model, train, _, (w, res, host) = worker_run
    _check(w, res, host, _host_train_traces(model, train))


def test_coverage_worker_numpy_inputs_give_the_same_results(worker_run):
    model, train, sets, (_, res, _) = worker_run
    _, res_np, _ = _run(model, train, sets, as_numpy=True)
    for ds in sets:
        for part in (1, 2):
            for name in NAMES:
                a, b = res[ds][part][name], res_np[ds][part][name]
                assert a.dtype == b.dtype and np.array_equal(a, b), (ds, part, name)


def test_coverage_worker_with_a_host_model(worker_run):
    model, train, sets, _ = worker_run
    host_model = copy.deepcopy(model).cpu()
    w, res, host = _run(host_model, train, sets, as_numpy=True)
    _check(w, res, host, _host_train_traces(host_model, train))


def test_coverage_worker_rejects_empty_sets_before_any_launch(worker_run):
    torch = _torch()
    from simple_tip_b200 import _lib
    from simple_tip_b200.core.coverage_worker import CoverageWorker

    model, train, _, (w, _, _) = worker_run
    before = _lib.launch_count()
    for empty in (np.zeros((0, 1, 12, 12), f32), torch.zeros((0, 1, 12, 12)).cuda()):
        with pytest.raises(ValueError):
            w.evaluate_all(empty)
        with pytest.raises(ValueError):
            CoverageWorker(model, NC_LAYERS, empty)
    assert _lib.launch_count() == before


def test_coverage_arm_result_files(worker_run, tmp_path):
    from simple_tip_b200.core import results as R
    from simple_tip_b200.core.apfd import apfd_from_order

    _, _, _, (w, res, host) = worker_run
    out = str(tmp_path)
    rng = np.random.default_rng(5)
    mis = {ds: rng.random(host[ds][0].shape[0]) < 0.3 for ds in res}
    for ds, m in mis.items():
        R.persist(out, "toy", ds, "is_misclassified", 0, m)
        times, scores, orders = res[ds]
        for name in w.metrics:
            R.persist_tip(out, "toy", ds, 0, name, scores[name], orders[name], times[name])
    for ds, m in mis.items():
        apfd = R.load_apfd_values(out, "toy", ds)
        times, scores, _ = res[ds]
        for name, metric in w.metrics.items():
            want_s, want_p = metric(host[ds])
            assert apfd[name][0] == apfd_from_order(m, np.argsort(-want_s))
            assert apfd[name + "-cam"][0] == apfd_from_order(m, np_oracle.cam_oracle(want_s, want_p))
            assert R.load_times(out, "toy", ds, 0, name) == times[name]


def test_single_model_paths_never_run_the_stack_kernels(monkeypatch):
    """One model's head sampler runs `engine.mc_head` and its coverage arm `prioritizers.cam_from_bits`, never their
    stacked forms with M = 1."""
    torch = _torch()
    from simple_tip_b200 import engine as E
    from simple_tip_b200.case_studies import mnist
    from simple_tip_b200.core import prioritizers as P
    from simple_tip_b200.core.activations import get_pred_and_uncertainty
    from simple_tip_b200.core.coverage_worker import CoverageWorker

    calls = []

    def spy(name, fn):
        def wrapped(*args, **kwargs):
            calls.append(name)
            return fn(*args, **kwargs)
        monkeypatch.setattr(E if name.startswith("mc_") else P, name, wrapped)
    for name in ("mc_head", "mc_head_stack"):
        spy(name, getattr(E, name))
    for name in ("cam_from_bits", "cam_from_bits_stack"):
        spy(name, getattr(P, name))
    torch.manual_seed(0)
    model = mnist.network().cuda()
    x = torch.rand(300, 28, 28, 1, device="cuda")
    get_pred_and_uncertainty(model, x, batch_size=128, sample_size=8, sampler="head")
    assert calls == ["mc_head"]
    calls.clear()
    CoverageWorker(model, mnist.NC_ACTIVATION_LAYERS, x, batch_size=BATCH).evaluate_all(x[:200])
    assert calls == ["cam_from_bits"] * len(NAMES)
