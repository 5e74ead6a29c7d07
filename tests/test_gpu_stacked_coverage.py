"""The coverage arm of a model stack on the GPU: tip_cam_bits_stack against one tip_cam_bits call per model (order and
state, exactly) and the dense-profile oracle, cam_from_bits_stack against cam_from_bits, the stacked coverage worker
against the single-model statistics, metrics and CAM on the stack's own traces, and a stacked-coverage prioritization
run against the sequential one."""
import os
import pickle
import shutil

import numpy as np
import pytest
import torch

from oracle import coverage_oracle as CO
from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E
from simple_tip_b200.case_studies import imdb, mnist
from simple_tip_b200.case_studies.stacked import stack
from simple_tip_b200.core import activations as A
from simple_tip_b200.core.aggregate_statistics import AggregateStatisticsCollector
from simple_tip_b200.core.coverage_worker import StackedCoverageWorker
from simple_tip_b200.core.neuron_coverage import KMNC, NAC, NBC, SNAC, TKNC, _score_dtype
from simple_tip_b200.core.prioritizers import cam_from_bits, cam_from_bits_stack

pytestmark = pytest.mark.gpu


# ---- the kernel -------------------------------------------------------------------------------------------------------------
def _profiles(models, n, words, seed):
    """Seeded bit profiles [M, n, words]: per model its own density (1/8 of the bits of a kept word), model 0 empty when
    there are several models."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 2 ** 32, size=(3, models, n, words), dtype=np.uint32)
    bits = r[0] & r[1] & r[2]
    keep = rng.random((models, n, words)) < rng.uniform(0.01, 0.3, size=(models, 1, 1))
    bits = np.where(keep, bits, 0).astype(np.uint32)
    if models > 1:
        bits[0] = 0
    return bits


def _run_single(bits, rounds, init_gain):
    """tip_cam_bits on one model's [n, words] profile until it is done: (order [n], state [4])."""
    lib = _lib.load()
    n, words = bits.shape
    gain = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    if not init_gain:
        gain = _popcounts(bits)
    covered = torch.zeros(2 * words, dtype=torch.int32, device="cuda")
    cand = torch.zeros(4 * _lib.CAM_MAX_BLOCKS, dtype=torch.int32, device="cuda")
    order = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    state = torch.zeros(4, dtype=torch.int32, device="cuda")
    first = init_gain
    while True:
        _lib.check(lib.tip_cam_bits(E._p(bits), n, words, E._p(gain), E._p(covered), E._p(cand), E._p(order),
                                    E._p(state), rounds, first, E._stream()), "tip_cam_bits")
        first = 0
        st = state.cpu().numpy()
        if st[1] or st[0] >= n:
            return order.cpu().numpy(), st


def _popcounts(bits):
    """row popcounts of an int32 profile [..., words] as int32, computed by torch"""
    b = bits.to(torch.int64) & 0xFFFFFFFF
    cnt = torch.zeros(b.shape[:-1], dtype=torch.int64, device=b.device)
    for k in range(32):
        cnt += ((b >> k) & 1).sum(dim=-1)
    return cnt.to(torch.int32).contiguous()


def _run_stack(bits, rounds, init_gain):
    """tip_cam_bits_stack on [M, n, words] until every model is done: (order [M, n], state [M, 4], launches)."""
    lib = _lib.load()
    models, n, words = bits.shape
    gain = torch.full((models, n), -7, dtype=torch.int32, device="cuda") if init_gain else _popcounts(bits)
    covered = torch.zeros((models, 2 * words), dtype=torch.int32, device="cuda")
    cand = torch.zeros(4 * _lib.CAM_MAX_BLOCKS, dtype=torch.int32, device="cuda")
    order = torch.full((models, n), -7, dtype=torch.int32, device="cuda")
    state = torch.zeros((models, 4), dtype=torch.int32, device="cuda")
    first, calls = init_gain, 0
    while True:
        _lib.check(lib.tip_cam_bits_stack(E._p(bits), models, n, words, E._p(gain), E._p(covered), E._p(cand),
                                          E._p(order), E._p(state), rounds, first, E._stream()), "tip_cam_bits_stack")
        first, calls = 0, calls + 1
        st = state.cpu().numpy()
        if not np.any((st[:, 1] == 0) & (st[:, 0] < n)):
            return order.cpu().numpy(), st, calls


def _check_against_single(bits_np, rounds, init_gain=1):
    bits = torch.from_numpy(bits_np.view(np.int32)).cuda()
    order, state, calls = _run_stack(bits, rounds, init_gain)
    for m in range(bits.shape[0]):
        want_order, want_state = _run_single(bits[m].contiguous(), rounds, init_gain)
        assert np.array_equal(order[m], want_order), (m, order[m][:8].tolist(), want_order[:8].tolist())
        assert np.array_equal(state[m], want_state), (m, state[m].tolist(), want_state.tolist())
    return order, state, calls


# (models, n, words)
SHAPES = [(1, 67, 37), (1, 5000, 1140), (3, 1, 1), (3, 67, 1140), (3, 5000, 37), (8, 1, 37), (8, 67, 1),
          (8, 5000, 1140), (40, 67, 37), (40, 1, 1140), (40, 5000, 1)]


@pytest.mark.parametrize("models, n, words", SHAPES)
def test_slices_equal_tip_cam_bits_per_model(models, n, words):
    bits = _profiles(models, n, words, seed=models * 7919 + n + words)
    order, state, _ = _check_against_single(bits, 4096)
    if models > 1:
        assert state[0, 0] == 0 and state[0, 1] == 1                 # the empty profile: no pick, done at once
    if n > 1:
        assert state[:, 0].max() > 1


@pytest.mark.parametrize("init_gain", [0, 1])
@pytest.mark.parametrize("models, n, words", [(3, 67, 37), (8, 5000, 37)])
def test_resumed_launches_of_two_rounds(models, n, words, init_gain):
    bits = _profiles(models, n, words, seed=n + init_gain)
    _, state, calls = _check_against_single(bits, 2, init_gain)
    assert calls > 2 and state[:, 0].max() > 4                       # the loop continued across many launches


def test_a_pick_with_more_than_4096_new_words():
    """model 1's first pick covers 4999 of 5000 words, its second then the last one; model 2's picks stay sparse"""
    models, n, words = 3, 67, 5000
    bits = _profiles(models, n, words, seed=3)
    bits[1, 20] = 0xFFFF
    bits[1, 20, 17] = 0
    bits[1, 40, 17] = 0xF0F0F0F0
    order, state, _ = _check_against_single(bits, 4096)
    assert order[1, 0] == 20 and state[1, 0] >= 2


def test_more_models_than_the_co_resident_grid():
    """300 small models: consecutive launches of the kernel, each with its own models' state"""
    bits = _profiles(300, 67, 4, seed=11)
    _, state, _ = _check_against_single(bits, 4096)
    assert (state[1:, 0] > 0).all()
    _check_against_single(bits[:290], 2)


@pytest.mark.parametrize("models, n, f", [(3, 50, 200), (8, 300, 1000), (40, 67, 96)])
def test_greedy_picks_equal_the_dense_oracle(models, n, f):
    rng = np.random.default_rng(n + f)
    prof = rng.random((models, n, f)) < rng.uniform(0.005, 0.1, size=(models, 1, 1))
    prof[0] = False
    prof[-1, 7] = True
    bits = torch.from_numpy(np.stack([CO.pack_plain(p) for p in prof]).view(np.int32)).cuda()
    order, state, _ = _run_stack(bits, 4096, 1)
    for m in range(models):
        want = CO.cam_greedy(prof[m])
        assert state[m, 0] == want.shape[0] and np.array_equal(order[m, :state[m, 0]], want), m


# ---- the host CAM -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("models, n, words, rounds", [(1, 500, 40, 4096), (5, 2000, 40, 4096), (5, 300, 3, 2),
                                                      (9, 1, 1, 4096)])
def test_cam_from_bits_stack_equals_cam_from_bits(models, n, words, rounds):
    bits_np = _profiles(models, n, words, seed=n * models)
    bits = torch.from_numpy(bits_np.view(np.int32)).cuda()
    rng = np.random.default_rng(models)
    scores = [rng.integers(0, 4, size=n).astype(np.int16) for _ in range(models)]       # many ties in the host tail
    kept = [s.copy() for s in scores]
    got = cam_from_bits_stack(scores, bits, rounds_per_launch=rounds)
    assert len(got) == models
    for m in range(models):
        want = np.array(list(cam_from_bits(scores[m], bits[m], rounds_per_launch=rounds)), dtype=np.int64)
        assert got[m].dtype == np.int64 and np.array_equal(got[m], want), m
        assert np.array_equal(scores[m], kept[m])                    # the caller's scores are not touched
    assert cam_from_bits_stack([], bits[:0]) == []


# ---- the worker against the single-model metrics on the stack's own traces ------------------------------------------------
def _networks(module, count, seed):
    torch.manual_seed(seed)
    return [module.network().cuda().eval() for _ in range(count)]


def _inputs(name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "mnist":
        return torch.from_numpy(rng.random((n, 28, 28, 1), dtype=np.float32)).cuda()
    return torch.from_numpy(rng.integers(0, 2000, size=(n, 100)).astype(np.int32)).cuda()


def _own_traces(net, layers, x, batch_size):
    """The stack's hooked layers, badge by badge, model-major: per badge a list of [M, b, *layer shape] tensors."""
    tm = A.TransparentModel(net, layers, include_last_layer=False)
    m = len(net.sources)
    return [[net.model_major(c, a) for c, a in zip(layers, tm.get_activations(net.stack_inputs([x[s:s + batch_size]] * m)))]
            for s in range(0, x.shape[0], batch_size)]


@pytest.mark.parametrize("name, module", [("mnist", mnist), ("imdb", imdb)])
def test_worker_equals_the_single_model_metrics_on_the_stacks_own_traces(name, module):
    models, batch = 3, 128
    net = stack(_networks(module, models, 5)).eval()
    assert net.channels_interleaved == (name == "mnist")
    layers = module.NC_ACTIVATION_LAYERS
    x_train, x_test = _inputs(name, 700, 1), _inputs(name, 300, 2)
    worker = StackedCoverageWorker(net, layers, x_train, batch_size=batch)
    results = worker.evaluate_all(x_test)
    assert len(results) == models
    train = _own_traces(net, layers, x_train, batch)
    test = _own_traces(net, layers, x_test, batch)
    for m in range(models):
        col = AggregateStatisticsCollector()
        for badge in train:
            col.track([a[m] for a in badge])
        mins, maxs, stds = col.get()
        for got, want in ((worker.mins[m], mins), (worker.maxs[m], maxs), (worker.stds[m], stds)):
            assert all(g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g, w, equal_nan=True)
                       for g, w in zip(got, want)), m
        per_layer = [torch.cat([badge[k][m] for badge in test]) for k in range(len(layers))]
        flat = torch.cat([l.reshape(l.shape[0], -1) for l in per_layer], dim=1).contiguous()
        d = int(flat.shape[1])
        words = int(_lib.load().tip_cover_packed_words(d))
        metrics = {**{f"NBC_{s}": NBC(mins, maxs, stds, s) for s in (0, 0.5, 1)},
                   **{f"SNAC_{s}": SNAC(maxs, stds, s) for s in (0, 0.5, 1)},
                   "NAC_0": NAC(0.0), "NAC_0.75": NAC(0.75), **{f"TKNC_{k}": TKNC(k) for k in (1, 2, 3)},
                   "KMNC_2": KMNC(mins, maxs, 2)}
        times, scores, orders = results[m]
        assert list(times) == list(scores) == list(orders) == list(metrics)
        for metric_id, metric in metrics.items():
            s, bits = metric.packed(per_layer if isinstance(metric, TKNC) else flat)
            s = s.cpu().numpy().astype(_score_dtype(d * (int(bits.shape[1]) // words)))
            assert scores[metric_id].dtype == s.dtype and np.array_equal(scores[metric_id], s), (m, metric_id)
            want = np.array(list(cam_from_bits(s, bits)), dtype=np.int64)
            assert np.array_equal(orders[metric_id], want), (m, metric_id)
            assert len(times[metric_id]) == 4 and times[metric_id] == results[0][0][metric_id], (m, metric_id)


# ---- the prioritization run ------------------------------------------------------------------------------------------------
def _blocks(rng, n):
    """MNIST-shaped uint8 images whose class is the 7 x 7 block (of a 4 x 4 grid) that is bright."""
    labels = rng.integers(0, 10, size=n)
    x = rng.integers(0, 90, size=(n, 28, 28), dtype=np.uint8)
    for i, c in enumerate(labels):
        r, k = divmod(int(c), 4)
        x[i, 7 * r:7 * r + 7, 7 * k:7 * k + 7] += np.uint8(160)
    return x, labels.astype(np.uint8)


APFD_TOLERANCE = 0.02       # as the stacked fault predictors': stacked against per-model forwards
COVERAGE = ("NBC_", "SNAC_", "NAC_", "TKNC_", "KMNC_")


@pytest.fixture(scope="module")
def prio_runs(tmp_path_factory):
    mp = pytest.MonkeyPatch()
    for k, v in {"B200TIP_KDE": "device", "B200TIP_COV": "device", "B200TIP_GMM": "device",
                 "B200TIP_KMEANS": "device", "B200TIP_MC": "head"}.items():
        mp.setenv(k, v)
    try:
        rng = np.random.default_rng(2)
        nominal = (_blocks(rng, 1200), _blocks(rng, 200))
        data = tmp_path_factory.mktemp("datasets")
        cx, cl = _blocks(rng, 200)
        np.save(data / "mnist_c_images.npy", np.expand_dims(255 - cx, -1))
        np.save(data / "mnist_c_labels.npy", cl.astype(np.int64))
        datasets = mnist.load_datasets(nominal, str(data))
        out = str(tmp_path_factory.mktemp("assets"))
        cs = mnist.MnistCaseStudy(out, datasets, epochs=1)
        np.random.seed(0)
        cs.train([0, 1, 2], stacked=True)
        res = {}
        for stacked in (False, True):
            cs.output_folder = str(tmp_path_factory.mktemp(f"prio_{stacked}"))
            os.makedirs(os.path.dirname(cs.model_path(0)))
            for i in (0, 1, 2):
                shutil.copyfile(os.path.join(out, "models", "mnist", f"model_{i}.pt"), cs.model_path(i))
            np.random.seed(5)
            res[stacked] = (cs.run_prio_eval([0, 1, 2], stacked=stacked, stack_size=2 if stacked else None,
                                             stacked_coverage=stacked), cs.output_folder)
    finally:
        mp.undo()
    return res


def _metric(f):
    """the approach a priorities file belongs to: mnist_<ds>_<id>_<approach>_<scores|cam_order>.npy"""
    return f.split("_", 3)[3]


def test_stacked_coverage_writes_the_sequential_files(prio_runs):
    (seq, seq_dir), (stk, stk_dir) = prio_runs[False], prio_runs[True]
    for sub in ("priorities", "times"):
        assert sorted(os.listdir(os.path.join(seq_dir, sub))) == sorted(os.listdir(os.path.join(stk_dir, sub)))
    files = sorted(os.listdir(os.path.join(seq_dir, "priorities")))
    assert sum(_metric(f).startswith(COVERAGE) for f in files) == 2 * 3 * 2 * 12
    fault_predictors = ("is_misclassified", "uncertainty_")
    for f in files:
        if any(k in f for k in fault_predictors) or _metric(f).startswith(COVERAGE):
            continue
        a, b = (np.load(os.path.join(d, "priorities", f)) for d in (seq_dir, stk_dir))
        np.testing.assert_array_equal(a, b, err_msg=f)
    assert list(seq) == list(stk) == [0, 1, 2]
    for model_id in seq:
        for ds in ("nominal", "ood"):
            assert list(seq[model_id][ds]) == list(stk[model_id][ds])
            for approach, apfd in seq[model_id][ds].items():
                if approach in ("softmax", "pcs", "softmax_entropy", "deep_gini", "VR") or approach.startswith(COVERAGE):
                    assert abs(apfd - stk[model_id][ds][approach]) <= APFD_TOLERANCE, (model_id, ds, approach, apfd,
                                                                                       stk[model_id][ds][approach])
                else:
                    assert apfd == stk[model_id][ds][approach], (model_id, ds, approach)


def test_stacked_coverage_time_files_hold_the_split_times(prio_runs):
    _, stk_dir = prio_runs[True]

    def load(ds, model_id, metric):
        with open(os.path.join(stk_dir, "times", f"mnist_{ds}_{model_id}_{metric}"), "rb") as f:
            return pickle.load(f)

    for ds in ("nominal", "ood"):
        for metric in ("NBC_0", "NAC_0.75", "TKNC_2", "KMNC_2"):
            first, second, alone = (load(ds, i, metric) for i in (0, 1, 2))
            assert len(first) == 4 and all(t >= 0 for t in first)
            assert first == second                                   # one stack of two: each holds half of every phase
            assert len(alone) == 4
