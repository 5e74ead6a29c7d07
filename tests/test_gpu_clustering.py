"""GPU tests of the device k-means discriminator: silhouette against sklearn, k-means quality and
determinism, predict, and the reference's k-means MultiModalSA test on the device backend."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _blobs(n, d, k, seed, spread=4.0, dtype=np.float64):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(k, d)) * spread
    lab = rng.integers(0, k, size=n)
    return (centres[lab] + rng.normal(size=(n, d))).astype(dtype), lab


def _sil_case(d, dtype, k, seed, n=1200):
    x, _ = _blobs(n, d, k, seed, spread=1.5, dtype=dtype)
    labels = np.random.default_rng(seed + 1).integers(0, k, size=n)
    labels[np.argsort(x[:, 0])[: n // 3]] = 0            # clusters that mean something, plus random mixing
    return x, labels


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 10, 96, 97, 300])
def test_silhouette_matches_sklearn(d, dtype):
    from sklearn import metrics

    from simple_tip_b200.core import clustering

    # d = 1: near neighbours' distances come out of an |x|^2 + |y|^2 - 2<x, y> cancellation with nothing to average
    # it over; the bound follows DESIGN.md §4b (measured on an H100: 1.4e-4 per row, 4e-6 on the score)
    row_tol = 5e-4 if d == 1 else 1e-4
    for k in range(2, 9):
        x, labels = _sil_case(d, dtype, k, seed=100 * d + k)
        want = metrics.silhouette_samples(x, labels)
        got = clustering.silhouette_samples(x, labels)
        assert got.dtype == np.float64 and got.shape == want.shape
        assert np.max(np.abs(got - want)) <= row_tol, (k, np.max(np.abs(got - want)))
        assert abs(clustering.silhouette_score(x, labels) - metrics.silhouette_score(x, labels)) <= 1e-5


@pytest.mark.parametrize("d", [16, 130])
def test_silhouette_singleton_cluster_and_label_values(d):
    from sklearn import metrics

    from simple_tip_b200.core import clustering

    x, labels = _sil_case(d, np.float32, 3, seed=7, n=700)
    labels = np.where(labels == 2, 11, labels)           # arbitrary label values
    labels[5] = -4                                       # a singleton cluster
    want = metrics.silhouette_samples(x, labels)
    got = clustering.silhouette_samples(x, labels)
    assert got[5] == 0.0
    assert np.max(np.abs(got - want)) <= 1e-4
    assert abs(clustering.silhouette_score(x, labels) - metrics.silhouette_score(x, labels)) <= 1e-5


@pytest.mark.parametrize("d", [32, 200])
def test_silhouette_with_heavy_row_duplication(d):
    from sklearn import metrics

    from simple_tip_b200.core import clustering

    base, lab = _blobs(60, d, 3, seed=3, spread=2.0, dtype=np.float32)
    x = np.repeat(base, 25, axis=0)                      # every row 25 times
    labels = np.repeat(lab, 25)
    want = metrics.silhouette_samples(x, labels)
    got = clustering.silhouette_samples(x, labels)
    # a duplicate's distance is the fp32 accumulator's cancellation noise instead of 0, and here every row has 24
    # of them: DESIGN.md §4b (measured on an H100: 1.0e-4 per row, 4.5e-5 on the score at d = 200)
    assert np.max(np.abs(got - want)) <= 5e-4, np.max(np.abs(got - want))
    assert abs(clustering.silhouette_score(x, labels) - metrics.silhouette_score(x, labels)) <= 2e-4


def test_silhouette_label_count_errors():
    from simple_tip_b200.core import clustering

    x = np.random.default_rng(0).normal(size=(10, 3))
    with pytest.raises(ValueError, match="Number of labels is 1. Valid values are 2 to n_samples - 1"):
        clustering.silhouette_score(x, np.zeros(10, dtype=int))
    with pytest.raises(ValueError, match="Number of labels is 10"):
        clustering.silhouette_samples(x, np.arange(10))


def test_silhouette_of_a_cuda_tensor_stays_on_the_device():
    import torch
    from sklearn import metrics

    from simple_tip_b200.core import clustering

    x, labels = _sil_case(20, np.float32, 4, seed=5, n=500)
    got = clustering.silhouette_samples(torch.from_numpy(x).cuda(), torch.from_numpy(labels).cuda())
    assert isinstance(got, torch.Tensor) and got.is_cuda
    assert np.max(np.abs(got.cpu().numpy() - metrics.silhouette_samples(x, labels))) <= 1e-4


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kmeans_finds_sklearns_optimum_on_separated_blobs(dtype):
    from sklearn.cluster import KMeans as SkKMeans

    from simple_tip_b200.core.clustering import KMeans

    x, _ = _blobs(3000, 24, 5, seed=11, spread=6.0, dtype=dtype)
    km = KMeans(5, n_init=10, random_state=0).fit(x)
    sk = SkKMeans(5, n_init=10, random_state=0).fit(x)
    assert km.cluster_centers_.dtype == dtype and km.labels_.dtype == np.int32
    key = lambda c: c[np.lexsort(c.T[::-1])]
    np.testing.assert_allclose(key(km.cluster_centers_), key(sk.cluster_centers_), atol=1e-4, rtol=0)
    assert km.inertia_ <= sk.inertia_ * (1 + 1e-6)
    assert 1 <= km.n_iter_ <= 300


def _near_tie_free(x, centres, labels):
    d2 = ((x.astype(np.float64)[:, None, :] - centres.astype(np.float64)[None]) ** 2).sum(-1)
    best = np.argmin(d2, axis=1)
    srt = np.sort(d2, axis=1)
    clear = (srt[:, 1] - srt[:, 0]) > 1e-5 * (1 + srt[:, 0])
    return best, clear


def test_kmeans_fixed_point_labels_and_centres():
    from simple_tip_b200.core.clustering import KMeans

    x, _ = _blobs(2000, 12, 4, seed=12, spread=3.0)
    km = KMeans(4, n_init=4, max_iter=300, tol=0.0, random_state=3).fit(x)   # tol 0: strict convergence
    best, clear = _near_tie_free(x, km.cluster_centers_, km.labels_)
    assert np.array_equal(km.labels_[clear], best[clear])
    for c in range(4):
        np.testing.assert_allclose(km.cluster_centers_[c], x[km.labels_ == c].mean(axis=0), rtol=0, atol=1e-12)


def test_kmeans_on_duplicated_rows_keeps_every_cluster():
    from simple_tip_b200.core.clustering import KMeans

    base, _ = _blobs(12, 6, 3, seed=13)
    x = np.repeat(base, 50, axis=0)
    for k in (2, 5, 12):
        km = KMeans(k, n_init=3, random_state=1).fit(x)
        assert np.bincount(km.labels_, minlength=k).min() > 0, k


def test_kmeans_is_deterministic_and_input_kind_agnostic():
    import torch

    from simple_tip_b200.core.clustering import KMeans

    x, _ = _blobs(5000, 40, 6, seed=14, spread=1.0, dtype=np.float32)
    a = KMeans(6, random_state=7).fit(x)
    b = KMeans(6, random_state=7).fit(x)
    t = KMeans(6, random_state=7).fit(torch.from_numpy(x).cuda())
    assert isinstance(t.cluster_centers_, torch.Tensor) and t.cluster_centers_.is_cuda
    for other in (b, t):
        oc = other.cluster_centers_
        oc = oc.cpu().numpy() if isinstance(oc, torch.Tensor) else oc
        ol = other.labels_.cpu().numpy() if isinstance(other.labels_, torch.Tensor) else other.labels_
        assert oc.tobytes() == a.cluster_centers_.tobytes()
        assert np.array_equal(ol, a.labels_)
        assert other.inertia_ == a.inertia_ and other.n_iter_ == a.n_iter_


def test_kmeans_predict_is_the_float64_argmin():
    from simple_tip_b200.core.clustering import KMeans

    x, _ = _blobs(3000, 30, 7, seed=15, spread=1.0, dtype=np.float32)
    km = KMeans(7, n_init=2, random_state=0).fit(x[:2000])
    q = x[2000:]
    got = km.predict(q)
    best, clear = _near_tie_free(q, km.cluster_centers_, got)
    assert clear.mean() > 0.99
    assert np.array_equal(got[clear], best[clear])


def test_k_means_clusterer_and_mmdsa_on_the_device():
    """The reference's tests/test_surprise.py::test_k_means_clusterer_and_mmdsa with backend="device"."""
    from simple_tip_b200.core.surprise import MDSA, MultiModalSA, _KmeansDiscriminator

    rng = np.random.RandomState(42)
    activations = np.concatenate([rng.random((100, 10)), rng.random((100, 10)) + 0.9])
    test_activations = np.array([[0.5] * 10, [1.4] * 10])
    discriminator = _KmeansDiscriminator(activations, [2, 3, 4], backend="device")
    assert discriminator.best_k == 2
    assert len(set(discriminator(test_activations, None))) == 2
    ood_data = test_activations + 2
    mmdsa = MultiModalSA.build_with_kmeans(activations, None, lambda x, _: MDSA(x), potential_k=[2, 3, 4],
                                           backend="device")
    assert np.all(mmdsa(ood_data, None) > mmdsa(test_activations, None))


def test_mmdsa_with_device_backend_scores_cuda_traces(monkeypatch):
    import torch

    from simple_tip_b200.core.surprise import MDSA, MultiModalSA

    monkeypatch.setenv("B200TIP_KMEANS", "device")
    rng = np.random.RandomState(1)
    train = np.concatenate([rng.random((300, 16)), rng.random((300, 16)) + 2.0])
    test = np.concatenate([rng.random((50, 16)), rng.random((50, 16)) + 2.0]) + 0.1
    mmdsa = MultiModalSA.build_with_kmeans(train, None, lambda x, _: MDSA(x), potential_k=[2, 3], subsampling=0.5)
    assert mmdsa.discriminator.backend == "device"
    host = mmdsa(test, None)
    dev = mmdsa(torch.from_numpy(test).cuda(), None)
    np.testing.assert_allclose(dev, host, rtol=1e-12, atol=0)
