"""GPU tests of the device k-means run by run: every run of tip_kmeans_fit against the float64 k-means++ / Lloyd
reference of oracle/kmeans_oracle.py, which uses the kernel's own draws.

Seeds (max_iter = 0) are compared bit for bit; after max_iter iterations each run's labels (one tip_kmeans_predict
pass over all runs), n_iter, centres and inertia.  A run is compared only when every decision along its trajectory
(draws, kept trials, nearest centres, relocated rows, the tol test) clears the device's rounding: 1e-9 relative for
float64 input; for float32 (distances are fp32 there, summed in warp order) four times the bound on an fp32 warp
sum's relative error.  At least 90% of the runs of a float64 case, and half of a float32 case, must qualify, so an
unlucky seed cannot quietly skip a case.
"""
import numpy as np
import pytest

from oracle import kmeans_oracle as KO

pytestmark = pytest.mark.gpu

SEED = 20261015


def _data(kind, n, d, seed, dtype):
    rng = np.random.default_rng(seed)
    if kind == "blobs":                                   # well separated: 64 centres far apart
        centres = rng.normal(size=(64, d)) * 8.0
        x = centres[rng.integers(0, 64, size=n)] + rng.normal(size=(n, d))
    elif kind == "overlap":                               # one Gaussian: many iterations, moving boundaries
        x = rng.normal(size=(n, d))
    elif kind == "offset":                                # a large common offset: cancellation in every difference
        x = 1e4 + rng.normal(size=(n, d)) * np.array([4.0, 1.0] * (d // 2) + [1.0] * (d % 2))
    elif kind == "equal":                                 # every row equal: the potential is 0 after the first seed
        x = np.full((n, d), 0.375)
    elif kind.startswith("repeat"):                       # m distinct rows (dyadic: exact sums), shuffled repeats
        m = int(kind[6:])
        base = rng.integers(-32, 32, size=(m, d)) / 8.0
        x = base[rng.permutation(np.arange(n) % m)]
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x.astype(dtype))


f32, f64 = np.float32, np.float64
# id, data, n, d, k, runs, dtype, tol, max_iter values
CASES = [
    ("n_eq_k_f64", "repeat64", 64, 8, 64, 10, f64, 1e-4, (0, 1, 300)),
    ("n_eq_k_grid_f32", "repeat7", 7, 3, 7, 10, f32, 1e-4, (0, 1, 300)),
    ("n9_d1", "overlap", 9, 1, 2, 64, f32, 0.0, (0, 1, 2, 300)),
    ("n9_k7_f64", "repeat9", 9, 2, 7, 10, f64, 1e-4, (0, 2, 300)),
    ("k1", "overlap", 500, 5, 1, 10, f64, 1e-4, (0, 1, 300)),
    ("odd_n_d65_f32", "blobs", 2037, 65, 3, 10, f32, 1e-4, (0, 1, 2, 300)),
    ("odd_n_d64_f64", "overlap", 1999, 64, 7, 10, f64, 0.0, (0, 2, 300)),
    ("n20000_d3_f64", "overlap", 20000, 3, 7, 10, f64, 1e-4, (0, 1, 300)),
    ("n20000_d3_f32", "blobs", 20000, 3, 2, 10, f32, 0.0, (0, 2, 300)),
    ("d300_k64_f64", "blobs", 3000, 300, 64, 1, f64, 1e-4, (0, 2, 300)),
    ("d2048_k2_runs10_f32", "blobs", 1200, 2048, 2, 10, f32, 1e-4, (0, 1, 300)),
    ("d2048_k64_runs10_f64", "blobs", 700, 2048, 64, 10, f64, 1e-4, (0, 2)),
    ("runs64_k2_f32", "overlap", 3000, 2, 2, 64, f32, 1e-4, (0, 300)),
    ("offset_f32", "offset", 1000, 16, 3, 10, f32, 1e-4, (0, 2, 300)),
    ("offset_f64", "offset", 3000, 16, 5, 10, f64, 0.0, (0, 2, 300)),
    ("equal_f32", "equal", 100, 4, 3, 10, f32, 1e-4, (0, 1, 300)),
    ("equal_f64", "equal", 33, 2, 7, 10, f64, 0.0, (0, 300)),
]
# duplicated rows with k = m, m + 1, 2m: the relocation corner (k > distinct rows leaves empty clusters)
DUP_CASES = [
    ("dup_k_eq_m_f64", "repeat12", 600, 6, 12, 10, f64, 1e-4, (1, 2, 300)),
    ("dup_k_m_plus_1_f64", "repeat12", 600, 6, 13, 10, f64, 1e-4, (1, 2, 300)),
    ("dup_k_2m_f32", "repeat12", 600, 6, 24, 10, f32, 0.0, (1, 2, 300)),
    ("dup_k_m_plus_1_f32", "repeat5", 97, 3, 6, 10, f32, 0.0, (1, 300)),
]


def _margin(dtype, d):
    """the relative error a decision must clear: float64 1e-9; float32: four times the bound on the relative error
    of an fp32 distance summed by one warp (ceil(d / 32) lane terms + 5 butterfly steps + 2 for each term) and so of
    every sum of such distances (potentials, cumulative sums), as the terms are positive"""
    return 1e-9 if dtype == f64 else 4 * (-(-d // 32) + 8) * 2.0 ** -24


def _device_fit(xd, k, runs, max_iter, tol_abs):
    """every run's centres, n_iter, final labels and inertia (tip_kmeans_fit + tip_kmeans_predict with runs)"""
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    lib = _lib.load()
    n, d = xd.shape
    dt = E.tip_dtype(xd.dtype)
    wb = int(lib.tip_kmeans_work_bytes(n, d, k, runs, dt))
    assert wb > 0
    work = torch.empty(wb, dtype=torch.uint8, device=xd.device)
    cen = torch.empty((runs, k, d), dtype=xd.dtype, device=xd.device)
    n_iter = torch.full((runs,), -1, dtype=torch.int32, device=xd.device)
    _lib.check(lib.tip_kmeans_fit(E._p(xd), dt, n, d, k, runs, max_iter, tol_abs, SEED, E._p(work), E._p(cen),
                                  E._p(n_iter), E._stream()), "tip_kmeans_fit")
    labels = torch.empty((runs, n), dtype=torch.int32, device=xd.device)
    sq = torch.empty((runs, n), dtype=torch.float64, device=xd.device)
    inertia = torch.empty(runs, dtype=torch.float64, device=xd.device)
    _lib.check(lib.tip_kmeans_predict(E._p(xd), dt, n, d, E._p(cen), k, runs, E._p(labels), E._p(sq), E._p(inertia),
                                      E._stream()), "tip_kmeans_predict")
    return cen.cpu().numpy(), n_iter.cpu().numpy(), labels.cpu().numpy(), inertia.cpu().numpy()


def _check_case(case, max_iter):
    import torch

    from simple_tip_b200 import engine as E

    name, kind, n, d, k, runs, dtype, tol, _ = case
    x = _data(kind, n, d, seed=n * 31 + d, dtype=dtype)
    xd = torch.from_numpy(x).cuda()
    # the absolute tol exactly as engine.kmeans_fit derives it
    tol_abs = float(torch.var(xd, dim=0, correction=0).mean()) * tol if tol > 0 else 0.0
    cen, n_iter, labels, inertia = _device_fit(xd, k, runs, max_iter, tol_abs)
    ref = KO.fit(x, k, runs, SEED, max_iter, tol_abs, dtype=dtype)
    thr = _margin(dtype, d)
    i_tol = 1e-12 if dtype == f64 else 1e-6
    scale = float(np.abs(x).max())
    compared, worst_c, worst_i = [], 0.0, 0.0
    for r in range(runs):
        s, run = ref.seedings[r], ref.runs[r]
        if min(s.margin, run.margin) <= thr:
            continue
        compared.append(r)
        where = f"{name} max_iter={max_iter} run {r}"
        if max_iter == 0:
            assert cen[r].tobytes() == x[s.idx].tobytes(), f"{where}: seeds differ from rows {s.idx.tolist()}"
        assert n_iter[r] == run.n_iter, (where, int(n_iter[r]), run.n_iter, run.stop)
        assert np.array_equal(labels[r], run.labels), (where, int(np.sum(labels[r] != run.labels)))
        want = run.centres
        err = np.abs(cen[r].astype(np.float64) - want)
        if dtype == f64:
            bound = 1e-12 * np.maximum(np.abs(want), scale)
        else:
            bound = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        assert np.all(err <= bound), (where, float(np.max(err - bound)))
        worst_c = max(worst_c, float(np.max(err / np.maximum(np.abs(want), scale))))
        ie = abs(inertia[r] - run.inertia) / max(run.inertia, 1e-300) if run.inertia > 0 else abs(inertia[r])
        assert ie <= i_tol, (where, inertia[r], run.inertia)
        worst_i = max(worst_i, ie)
    # float32 draws land within the fp32 error of a row boundary of the cumulative D^2 far more often (the bound
    # is ~1e-6 of the potential, and a seeding makes (k - 1) * trials draws), so half of the runs must qualify there
    need = 0.9 if dtype == f64 or KO.exact_grid(x) else 0.5
    assert len(compared) >= max(1, need * runs), (name, max_iter, f"only {len(compared)} of {runs} runs clear the margin")

    # the best run: engine.kmeans_fit (and KMeans) keep the first run of lowest device inertia, the oracle's pick
    cb, lb, ib, itb = E.kmeans_fit(xd, k, runs, max_iter, tol, SEED)
    r_dev = next(r for r in range(runs) if cen[r].tobytes() == cb.cpu().numpy().tobytes())
    assert ib == inertia[r_dev] == inertia.min() and itb == n_iter[r_dev]
    oi = ref.inertia
    others = np.delete(oi, ref.best)
    clear = others.size == 0 or np.min(np.abs(others - oi[ref.best])) > 10 * i_tol * max(oi[ref.best], 1e-300)
    if clear and len(compared) == runs:
        assert r_dev == ref.best, (name, max_iter, r_dev, ref.best)
    else:   # runs that reach the same clustering tie up to rounding: the pick must be one of them
        assert oi[r_dev] <= oi.min() * (1 + 10 * i_tol) + 1e-300, (name, max_iter, r_dev, ref.best)
    if max_iter >= 1:
        from simple_tip_b200.core.clustering import KMeans

        km = KMeans(k, n_init=runs, max_iter=max_iter, tol=tol, random_state=SEED).fit(x)
        assert km.cluster_centers_.tobytes() == cen[r_dev].tobytes() and km.inertia_ == ib and km.n_iter_ == itb
    print(f"[kmeans-ref] {name} max_iter={max_iter}: {len(compared)}/{runs} runs compared exactly, "
          f"worst centre err {worst_c:.3g} (rel. to max(|c|, |x|max)), worst inertia err {worst_i:.3g}, "
          f"n_iter {sorted(set(n_iter.tolist()))}")


def _params(cases):
    return [pytest.param(c, m, id=f"{c[0]}-it{m}") for c in cases for m in c[8]]


@pytest.mark.parametrize("case, max_iter", _params(CASES))
def test_every_run_matches_the_reference(case, max_iter):
    _check_case(case, max_iter)


@pytest.mark.parametrize("case, max_iter", _params(DUP_CASES))
def test_every_run_matches_the_reference_on_duplicated_rows(case, max_iter):
    _check_case(case, max_iter)


def test_seeding_only_fit_returns_the_seeds():
    import torch

    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.clustering import KMeans

    x = _data("overlap", 300, 4, seed=1, dtype=f64)
    cen, lab, inertia, n_iter = E.kmeans_fit(torch.from_numpy(x).cuda(), 5, 3, 0, 1e-4, SEED)
    rows = {x[i].tobytes() for i in range(300)}
    assert n_iter == 0 and all(c.tobytes() in rows for c in cen.cpu().numpy())
    with pytest.raises(ValueError):
        KMeans(5, max_iter=0)
