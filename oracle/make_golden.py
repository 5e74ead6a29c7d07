"""Generates tests/golden/*.npz by running the UNMODIFIED reference classes
(/root/reference, via oracle/ref_harness.py) on small seeded inputs.

Run in the authoring container only:  python oracle/make_golden.py
The fixtures (inputs + reference outputs) are committed; the GPU box and CI never need
/root/reference.  Re-running must reproduce the committed files bit for bit (all inputs
come from seeded generators).
"""
from __future__ import annotations

import io
import os
import sys
import warnings
from contextlib import redirect_stdout

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from oracle import np_oracle, ref_harness  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def quiet(fn, *a, **k):
    with redirect_stdout(io.StringIO()), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def ref_dsa(ref, xtr, ytr, xte, pte, **kw):
    sa = quiet(ref.surprise.DSA, xtr, ytr, **kw)
    import tqdm

    real = tqdm.tqdm
    try:
        tqdm.tqdm = lambda it, **_: it          # silence the progress bar only
        dsa = quiet(sa, xte, pte)
    finally:
        tqdm.tqdm = real
    # per-class distances straight from the reference's _dsa_distances (surprise.py:615-631)
    da = np.zeros(xte.shape[0], dtype=sa.train_activations.dtype)
    db = np.zeros_like(da)
    for c in range(sa.num_classes):
        rows = np.argwhere(np.asarray(pte) == c).flatten()
        for chunk in np.array_split(rows, max(1, int(np.ceil(rows.size / 64)))):
            if chunk.size:
                a, b = sa._dsa_distances(np_oracle.flatten_rows(np.asarray(xte))[chunk], c)
                da[chunk], db[chunk] = a, b
    return dsa, da, db


def dsa_cases(ref):
    cases = {}
    # g1: float32 Gaussian clusters
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(600, 100, 16, 4, seed=11)
    cases["f32_clusters"] = (xtr, ytr, xte, pte, {})
    # g2: the reference's own plausibility inputs (tests/test_surprise.py:141-151), float64
    rng = np.random.RandomState(42)
    act = rng.random((100, 10))
    lab = rng.randint(0, 3, size=100)
    cases["f64_plausibility_id"] = (act, lab, act[:10], lab[:10], {})
    cases["f64_plausibility_ood"] = (act, lab, act[:10] + 10, lab[:10], {})
    # g3: exact ties — small-integer valued float32 traces, duplicated train rows
    rng = np.random.default_rng(12)
    base = rng.integers(0, 3, size=(60, 12)).astype(np.float32)
    xtr = np.concatenate([base, base[:20], base[5:25]])
    ytr = np.concatenate([np.arange(60) % 3, np.arange(20) % 3, (np.arange(20) + 5) % 3]).astype(np.int64)
    xte = np.concatenate([base[:15], rng.integers(0, 3, size=(25, 12)).astype(np.float32)])
    pte = rng.integers(0, 3, size=40).astype(np.int64)
    cases["f32_ties"] = (xtr, ytr, xte, pte, {})
    # g4: the study's configuration: subsampling=0.3 (handler_surprise.py:24)
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(1000, 64, 32, 5, seed=13)
    cases["f32_subsample"] = (xtr, ytr, xte, pte, {"subsampling": 0.3})
    # g5/g6: D > 128 (recursive pairwise split) and D < 8 (sequential sum)
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(300, 40, 300, 3, seed=14)
    cases["f32_d300"] = (xtr, ytr, xte, pte, {})
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(200, 30, 5, 2, seed=15)
    cases["f32_d5"] = (xtr, ytr, xte, pte, {})
    # g7: ragged — one class absent from the test predictions, badge_size 7, 3-D traces
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(240, 33, 24, 4, seed=16)
    pte[pte == 2] = 1
    cases["f32_ragged_3d"] = (xtr.reshape(240, 2, 12), ytr, xte.reshape(33, 2, 12), pte, {"badge_size": 7})
    out = {}
    for name, (xtr, ytr, xte, pte, kw) in cases.items():
        dsa, da, db = ref_dsa(ref, xtr, ytr, xte, pte, **kw)
        out[f"{name}.xtr"], out[f"{name}.ytr"], out[f"{name}.xte"], out[f"{name}.pte"] = xtr, ytr, xte, pte
        out[f"{name}.dsa"], out[f"{name}.dist_a"], out[f"{name}.dist_b"] = dsa, da, db
        out[f"{name}.kw"] = np.array(repr(kw))
    np.savez_compressed(os.path.join(OUT, "dsa_reference.npz"), **out)
    print("dsa:", list(cases))


def lsa_cases(ref):
    out = {}
    rng = np.random.RandomState(42)
    # the reference's plausibility inputs (tests/test_surprise.py:141-151): finite ID, inf OOD
    act = rng.random((100, 10))
    sa = quiet(ref.surprise.LSA, act)
    out["plaus.xtr"], out["plaus.xte"] = act, np.concatenate([act[:10], act[:10] + 10])
    out["plaus.lsa"] = quiet(sa, out["plaus.xte"])
    # unit cube 2000 x 10
    a = rng.random((2000, 10)).astype(np.float32)
    t = rng.random((100, 10)).astype(np.float32)
    out["cube.xtr"], out["cube.xte"] = a, t
    out["cube.lsa"] = quiet(quiet(ref.surprise.LSA, a), t)
    # clusters with column removal (max_features=30 of 40)
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(3000, 120, 40, 4, seed=21)
    sa = quiet(ref.surprise.LSA, xtr, max_features=30)
    out["mf30.xtr"], out["mf30.xte"] = xtr, xte
    out["mf30.lsa"] = quiet(sa, xte)
    out["mf30.removed"] = np.array(sa.removed_neurons, dtype=np.int64)
    # pc-lsa (MultiModalSA.build_by_class, handler_surprise.py:26)
    mm = quiet(ref.surprise.MultiModalSA.build_by_class, xtr, ytr, lambda x, y: ref.surprise.LSA(x))
    out["pclsa.ytr"], out["pclsa.pte"] = ytr, pte
    out["pclsa.lsa"] = quiet(mm, xte, pte)
    # singular covariance (duplicated column) -> _stabilize_covariance replaces the diagonal
    base = rng.random((500, 6))
    sing = np.concatenate([base, base[:, :1]], axis=1)
    sa = quiet(ref.surprise.LSA, sing)
    out["singular.xtr"], out["singular.xte"] = sing, sing[:20] + 0.01
    out["singular.lsa"] = quiet(sa, out["singular.xte"])
    out["singular.prepare_failed"] = np.array(bool(sa.kde.prepare_failed))
    # moderately far points: finite but large values (log-domain stress)
    out["far.xtr"], out["far.xte"] = a, (t * 3.0 + 0.5).astype(np.float32)
    out["far.lsa"] = quiet(quiet(ref.surprise.LSA, a), out["far.xte"])
    np.savez_compressed(os.path.join(OUT, "lsa_reference.npz"), **out)
    print("lsa: plaus cube mf30 pclsa singular far;",
          "inf count", int(np.isinf(out["plaus.lsa"]).sum()), int(np.isinf(out["far.lsa"]).sum()),
          "singular prepare_failed", bool(sa.kde.prepare_failed))


def coverage_cases(ref):
    out = {}
    rng = np.random.default_rng(31)
    for name, dt_act, dt_stat, sections, n, d in [
        ("k2_f32", np.float32, np.float32, 2, 17, 29),
        ("k10_f32", np.float32, np.float32, 10, 33, 64),
        ("k1000_f32", np.float32, np.float32, 1000, 9, 40),
        ("k7_f64stat", np.float32, np.float64, 7, 12, 21),
        ("k5_f64", np.float64, np.float64, 5, 10, 16),
    ]:
        stat = np.maximum(rng.normal(size=(200, d)), 0).astype(dt_stat)
        mins, maxs = stat.min(axis=0), stat.max(axis=0)
        maxs[::9] = mins[::9]                      # constant neurons: jumps == 0
        act = np.maximum(rng.normal(size=(n, d)) * 1.3, 0).astype(dt_act)
        act[0, 1] = maxs[1]                        # a == max hits no bucket (half-open)
        act[1, 2] = mins[2]                        # a == min hits bucket 0
        act[2, 3] = -0.5                           # below range
        # split into two "layers" like the handlers pass them (neuron_coverage.py:25-28)
        cut = d // 3
        km = ref.neuron_coverage.KMNC([mins[:cut], mins[cut:]], [maxs[:cut], maxs[cut:]], sections)
        score, prof = km([act[:, :cut], act[:, cut:]])
        out[f"{name}.mins"], out[f"{name}.maxs"], out[f"{name}.act"] = mins, maxs, act
        out[f"{name}.cut"], out[f"{name}.sections"] = np.array(cut), np.array(sections)
        out[f"{name}.score"] = score
        out[f"{name}.bucket"] = np.where(prof.any(axis=2), prof.argmax(axis=2), -1).astype(np.int32)
        out[f"{name}.hits"] = prof.sum(axis=2).astype(np.int32)
    np.savez_compressed(os.path.join(OUT, "kmnc_reference.npz"), **out)
    print("kmnc ok")


def gini_apfd_cases(ref):
    out = {}
    for name, dt in (("c1_f32", np.float32), ("c1_f64", np.float64)):
        p, truth = np_oracle.synth_softmax(2000, 10, seed=1, dtype=dt)
        pred, gini = ref.deepgini.DeepGini.calculate(p)
        order = np.argsort(-gini)                                  # eval_apfd_table.py:86
        fault = (pred != truth)
        out[f"{name}.p"], out[f"{name}.truth"] = p, truth
        out[f"{name}.pred"], out[f"{name}.gini"] = pred, gini
        out[f"{name}.apfd"] = np.array(ref.apfd.apfd_from_order(fault, order))
    p, _ = np_oracle.synth_softmax(64, 1000, seed=2, dtype=np.float32)   # wide rows: n > 128 path
    pred, gini = ref.deepgini.DeepGini.calculate(p)
    out["wide.p"], out["wide.pred"], out["wide.gini"] = p, pred, gini
    rng = np.random.default_rng(41)
    for i in range(4):
        n = int(rng.integers(5, 400))
        fault = rng.random(n) < 0.3
        fault[0] = True
        order = rng.permutation(n)
        out[f"apfd{i}.fault"], out[f"apfd{i}.order"] = fault, order
        out[f"apfd{i}.value"] = np.array(ref.apfd.apfd_from_order(fault, order))
    np.savez_compressed(os.path.join(OUT, "gini_apfd_reference.npz"), **out)
    print("gini/apfd ok")


def prioritizer_cases(ref):
    out = {}
    rng = np.random.default_rng(51)
    for i, (n, w, dens) in enumerate([(12, 9, 0.3), (40, 64, 0.1), (30, 20, 0.6), (25, 50, 0.0)]):
        prof = rng.random((n, w)) < dens
        scores = prof.sum(axis=1).astype(np.int64) if i % 2 == 0 else rng.random(n)
        out[f"cam{i}.profiles"], out[f"cam{i}.scores"] = prof, scores
        out[f"cam{i}.order"] = np.array(list(ref.prioritizers.cam(scores, prof.copy())), dtype=np.int64)
        out[f"cam{i}.ctm"] = np.array(list(ref.prioritizers.ctm(scores)), dtype=np.int64)
    m = ref.surprise.SurpriseCoverageMapper(10, 2.5)
    vals = rng.random(50) * 3
    out["scm.values"], out["scm.profile"] = vals, m.get_coverage_profile(vals)
    m = ref.surprise.SurpriseCoverageMapper(10, 2.5, overflow_bucket=True)
    out["scm.profile_overflow"] = m.get_coverage_profile(vals)
    np.savez_compressed(os.path.join(OUT, "prioritizers_reference.npz"), **out)
    print("prioritizers ok")


def cam_kmnc_cases(ref):
    """CAM over KMNC profiles (handler_coverage.py:122-124: `cam(scores, profiles)` with the dense
    N x D x k profile of neuron_coverage.py:82-94), stored with the COMPACT bucket ids so that a CAM
    that never materialises the dense profile can be checked against the reference's order."""
    out = {}
    for i, (n, d, k, seed) in enumerate([(40, 24, 5, 61), (120, 64, 16, 62), (300, 96, 50, 63), (64, 32, 2, 64)]):
        act, mins, maxs = np_oracle.synth_relu(n, d, seed=seed)
        km = ref.neuron_coverage.KMNC([mins], [maxs], k)
        score, prof = km([act])
        order = np.array(list(ref.prioritizers.cam(score, prof.copy())), dtype=np.int64)
        out[f"camk{i}.bucket"] = np.where(prof.any(axis=2), prof.argmax(axis=2), -1).astype(np.int32)
        out[f"camk{i}.score"], out[f"camk{i}.sections"], out[f"camk{i}.order"] = score, np.array(k), order
        assert int(prof.sum(axis=2).max()) <= 1
    np.savez_compressed(os.path.join(OUT, "cam_kmnc_reference.npz"), **out)
    print("cam over kmnc ok")


def sibling_cases(ref):
    """NAC / NBC / SNAC / TKNC (neuron_coverage.py:52-62,97-173) with the configurations of
    handler_coverage.py:49-101, fitted on statistics from the reference's own AggregateStatisticsCollector
    (welford==0.2.5 restated, see ref_harness), plus `cam` on each profile (handler_coverage.py:122-124) and the
    surprise-coverage CAM of handler_surprise.py:101-115."""
    agg = ref_harness.load_aggregate_statistics()
    nc = ref.neuron_coverage
    out = {}
    rng = np.random.default_rng(71)
    shapes = [(6, 5, 4), (37,), (3, 11)]                       # conv-like, dense, 2-D layers
    n_train, n_test = 230, 90

    def draw(n, scale):
        return [np.maximum(rng.normal(size=(n,) + sh) * scale + 0.2, 0).astype(np.float32) for sh in shapes]

    train = draw(n_train, 1.0)
    col = agg.AggregateStatisticsCollector()
    cuts = [0, 64, 128, 131, 230]                              # ragged badges, like the last batch of a dataset walk
    for a, b in zip(cuts[:-1], cuts[1:]):
        col.track([l[a:b] for l in train])
    mins, maxs, stds = col.get()
    test = draw(n_test, 1.4)
    test[1][0, 3] = maxs[1][3]                                 # exactly on a boundary (>= / <= matter)
    test[1][1, 4] = mins[1][4]
    for i, l in enumerate(train):
        out[f"sib.train{i}"] = l
    for i, l in enumerate(test):
        out[f"sib.test{i}"] = l
    out["sib.cuts"] = np.array(cuts)
    for i in range(len(shapes)):
        out[f"sib.min{i}"], out[f"sib.max{i}"], out[f"sib.std{i}"] = mins[i], maxs[i], stds[i]
    metrics = {"NAC_0": nc.NAC(0.0), "NAC_0.75": nc.NAC(0.75),
               "NBC_0": nc.NBC(mins, maxs, stds, 0), "NBC_0.5": nc.NBC(mins, maxs, stds, 0.5), "NBC_1": nc.NBC(mins, maxs, stds, 1),
               "SNAC_0": nc.SNAC(maxs, stds, 0), "SNAC_0.5": nc.SNAC(maxs, stds, 0.5), "SNAC_1": nc.SNAC(maxs, stds, 1),
               "TKNC_1": nc.TKNC(1), "TKNC_2": nc.TKNC(2), "TKNC_3": nc.TKNC(3)}
    for name, m in metrics.items():
        score, prof = m([l.copy() for l in test])
        out[f"sib.{name}.score"], out[f"sib.{name}.profile"] = score, prof
        out[f"sib.{name}.cam"] = np.array(list(ref.prioritizers.cam(score, prof.copy())), dtype=np.int64)
    # float64 activations / statistics
    tr64 = [l.astype(np.float64) for l in train[:2]]
    col = agg.AggregateStatisticsCollector()
    col.track(tr64)
    mn, mx, sd = col.get()
    te64 = [l.astype(np.float64) for l in test[:2]]
    for i in range(2):
        out[f"sib64.min{i}"], out[f"sib64.max{i}"], out[f"sib64.std{i}"] = mn[i], mx[i], sd[i]
    s, p = nc.NBC(mn, mx, sd, 0.5)(te64)
    out["sib64.NBC_0.5.score"], out["sib64.NBC_0.5.profile"] = s, p
    # surprise-coverage CAM: 1000 buckets up to the largest observed value (handler_surprise.py:101-115, NUM_SC_BUCKETS)
    sa = np.abs(rng.normal(size=400)) * 3
    sa[17] = sa.max()                                          # the maximum itself falls outside the half-open last bucket
    mapper = ref.surprise.SurpriseCoverageMapper(1000, np.max(sa))
    prof = mapper.get_coverage_profile(sa)
    out["sc.values"], out["sc.profile"] = sa, prof
    out["sc.cam"] = np.array(list(ref.prioritizers.cam(sa, prof.copy())), dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "siblings_reference.npz"), **out)
    print("siblings ok", {k: int(out[f"sib.{k}.score"].sum()) for k in metrics})


def coverage_edge_cases(ref):
    """The reference's TKNC at k <= 0 and k >= d (its slice `argsort(layer)[..., -k:]` marks every neuron for k = 0
    and all but the |k| lowest for k < 0) on tie-free layers, and its NAC on activations that are not float32 /
    float64 (`activations > threshold` compares in NumPy's promotion of the activation dtype with a Python float)."""
    nc = ref.neuron_coverage
    out = {}
    rng = np.random.default_rng(97)
    widths = (1, 5, 37)
    # a permutation per row: distinct values in every row, so the reference's unstable argsort has no ties to break
    layers = [(np.stack([rng.permutation(w) for _ in range(9)]) * 0.37 - 2).astype(np.float32) for w in widths]
    for i, l in enumerate(layers):
        out[f"tknc.layer{i}"] = l
    d = sum(widths)
    for k in (0, -1, -3, d, d + 2):
        score, prof = nc.TKNC(k)([l.copy() for l in layers])
        out[f"tknc.k{k}.score"], out[f"tknc.k{k}.profile"] = score, prof
    grid = np.array([0.3, 0.75, 1.9999999999, 2.0, 1.0, 0.0, -1.0]).astype(np.float16)   # and one float16 ulp either side
    acts = {
        "f16": np.concatenate([grid, np.nextafter(grid, np.float16(3)), np.nextafter(grid, np.float16(-3)),
                               rng.normal(size=11).astype(np.float16)]),
        "i16": np.array([-3, -1, 0, 1, 2, 3, 300, -300], dtype=np.int16),
        "u8": np.array([0, 1, 2, 3, 255], dtype=np.uint8),
        "bool": np.array([False, True]),
    }
    for name, a in acts.items():
        a = np.resize(a, 2 * a.size).reshape(2, -1)
        out[f"nac.{name}.act"] = a
        for t in (0.3, 0.75, 0.9999999999, 1.9999999999):
            score, prof = nc.NAC(t)([a.copy()])
            out[f"nac.{name}.{t!r}.score"], out[f"nac.{name}.{t!r}.profile"] = score, prof
    np.savez_compressed(os.path.join(OUT, "coverage_edges_reference.npz"), **out)
    print("coverage edges ok", {k: int(out[f"tknc.k{k}.score"][0]) for k in (0, -1, -3, d, d + 2)})


def mdsa_mlsa_cases(ref):
    """MDSA / MLSA (surprise.py:374-393,498-520) and their per-class forms (handler_surprise.py:28-33) run by the
    reference's own classes on top of this container's scikit-learn.  GaussianMixture's fit draws from NumPy's
    global RNG, so the fitted parameters are stored next to the outputs."""
    out = {}
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(3000, 400, 48, 4, seed=91, spread=1.5)
    xtr, xte = xtr.astype(np.float64), xte.astype(np.float64)
    out["x.xtr"], out["x.ytr"], out["x.xte"], out["x.pte"] = xtr, ytr, xte, pte
    m = quiet(ref.surprise.MDSA, xtr)
    out["mdsa.out"] = m(xte)
    out["mdsa.location"], out["mdsa.precision"] = m.covariance_matrix.location_, m.covariance_matrix.get_precision()
    pc = quiet(ref.surprise.MultiModalSA.build_by_class, xtr, ytr, lambda x, y: ref.surprise.MDSA(x))
    out["pcmdsa.out"] = pc(xte, pte)
    np.random.seed(1234)
    g = quiet(ref.surprise.MLSA, xtr, 3)
    out["mlsa.out"] = g(xte)
    out["mlsa.means"], out["mlsa.prec_chol"], out["mlsa.weights"] = g.gmm.means_, g.gmm.precisions_cholesky_, g.gmm.weights_
    # a rank-deficient covariance (duplicated column): sklearn's pinvh precision is singular
    xs = np.concatenate([xtr[:, :10], xtr[:, :1]], axis=1)
    ms = quiet(ref.surprise.MDSA, xs)
    out["sing.xtr"], out["sing.xte"] = xs, np.concatenate([xte[:, :10], xte[:, :1]], axis=1)
    out["sing.out"] = ms(out["sing.xte"])
    np.savez_compressed(os.path.join(OUT, "mdsa_mlsa_reference.npz"), **out)
    print("mdsa/mlsa ok", float(out["mdsa.out"].mean()), float(out["mlsa.out"].mean()))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    ref = ref_harness.load()
    if len(sys.argv) > 1 and sys.argv[1] == "cam_kmnc":      # add this file without touching the others
        cam_kmnc_cases(ref)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "mdsa_mlsa":
        mdsa_mlsa_cases(ref)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "siblings":
        sibling_cases(ref)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "coverage_edges":
        coverage_edge_cases(ref)
        sys.exit(0)
    dsa_cases(ref)
    lsa_cases(ref)
    coverage_cases(ref)
    gini_apfd_cases(ref)
    prioritizer_cases(ref)
    cam_kmnc_cases(ref)
    sibling_cases(ref)
    mdsa_mlsa_cases(ref)
    coverage_edge_cases(ref)
    print("sizes:", {f: os.path.getsize(os.path.join(OUT, f)) for f in sorted(os.listdir(OUT))})
