"""CPU tests of the device k-means discriminator's host side: backend selection, argument checks that run
before any launch, the silhouette work list and the export table of the new entry points."""
import numpy as np
import pytest

from simple_tip_b200 import _lib
from simple_tip_b200 import engine as E
from simple_tip_b200.core import clustering
from simple_tip_b200.core.surprise import MDSA, MultiModalSA, _KmeansDiscriminator


def _two_blobs():
    rng = np.random.RandomState(42)
    return np.concatenate([rng.random((40, 4)), rng.random((40, 4)) + 0.9])


def test_sklearn_backend_stays_the_default(monkeypatch):
    monkeypatch.delenv("B200TIP_KMEANS", raising=False)
    disc = _KmeansDiscriminator(_two_blobs(), [2, 3])
    assert disc.backend == "sklearn" and disc.best_k == 2
    assert type(disc.best_clusterer).__module__.startswith("sklearn")


def test_unknown_backend_is_rejected():
    with pytest.raises(ValueError, match="backend"):
        _KmeansDiscriminator(_two_blobs(), [2], backend="cpu")


def test_device_backend_without_a_gpu_fails_loudly(monkeypatch):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        _KmeansDiscriminator(_two_blobs(), [2], backend="device")
    monkeypatch.setenv("B200TIP_KMEANS", "device")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        MultiModalSA.build_with_kmeans(_two_blobs(), None, lambda x, _: MDSA(x), potential_k=[2])
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        clustering.silhouette_score(_two_blobs(), np.arange(80) % 2)


@pytest.mark.parametrize("k", [0, 65, 100])
def test_kmeans_rejects_k_outside_1_to_64_before_launching(k):
    with pytest.raises(ValueError, match="n_clusters"):
        clustering.KMeans(n_clusters=k)


@pytest.mark.parametrize("counts,span_tiles", [([300, 1, 700], 1), ([5, 5], 2), ([1000, 2000, 17, 3000], 2),
                                               ([129, 0, 257], 1)])
def test_silhouette_items_put_every_pair_in_one_slot_of_its_cluster(counts, span_tiles):
    counts = np.asarray(counts)
    off = np.concatenate(([0], np.cumsum(counts)))
    n = int(off[-1])
    items, slot_cluster = E.silhouette_items(counts, span_tiles)
    assert np.all(np.diff(slot_cluster) >= 0)
    hits = np.zeros((n, n), dtype=np.int32)
    slot_of = -np.ones((n, n), dtype=np.int64)
    for q0, nq, c0, c1, slot, flags in items:
        assert flags == 0 and 1 <= nq <= _lib.ROW_TILE
        cl = slot_cluster[slot]
        assert off[cl] <= c0 < c1 <= off[cl + 1], "a span crosses a cluster boundary"
        hits[q0:q0 + nq, c0:c1] += 1
        slot_of[q0:q0 + nq, c0:c1] = slot
    assert np.all(hits == 1)
    col_cluster = np.repeat(np.arange(len(counts)), counts)
    assert np.array_equal(slot_cluster[slot_of], np.broadcast_to(col_cluster, (n, n)))


def test_new_entry_points_are_declared_and_bound():
    names = {"tip_kmeans_work_bytes", "tip_kmeans_fit", "tip_kmeans_predict", "tip_sil_prep", "tip_sil_dsum",
             "tip_sil_finish"}
    assert names <= set(_lib.symbols())
    lib = _lib.load()
    for name in names:
        assert hasattr(lib, name)
