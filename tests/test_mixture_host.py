"""CPU tests of the device Gaussian-mixture backend's host side: backend selection, argument checks that run before
any launch, and the export table of the new entry points."""
import numpy as np
import pytest

from simple_tip_b200 import _lib
from simple_tip_b200.core import mixture
from simple_tip_b200.core.surprise import MLSA, MultiModalSA


def _blobs():
    rng = np.random.RandomState(42)
    return np.concatenate([rng.random((60, 3)), rng.random((60, 3)) + 0.9])


def test_sklearn_backend_stays_the_default(monkeypatch):
    monkeypatch.delenv("B200TIP_GMM", raising=False)
    m = MLSA(_blobs(), num_components=2)
    assert m.backend == "sklearn"
    assert type(m.gmm).__module__.startswith("sklearn")


def test_unknown_backend_is_rejected(monkeypatch):
    with pytest.raises(ValueError, match="backend"):
        MLSA(_blobs(), num_components=2, backend="cpu")
    monkeypatch.setenv("B200TIP_GMM", "cuda")
    with pytest.raises(ValueError, match="backend"):
        MLSA(_blobs(), num_components=2)


def test_device_backend_without_a_gpu_fails_loudly(monkeypatch):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        MLSA(_blobs(), num_components=2, backend="device")
    monkeypatch.setenv("B200TIP_GMM", "device")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        MultiModalSA.build_by_class(_blobs(), np.arange(120) % 2, lambda x, y: MLSA(x, num_components=3))
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        mixture.GaussianMixture(2).fit(_blobs())


@pytest.mark.parametrize("kw,match", [({"n_components": 0}, "n_components"), ({"n_components": 65}, "n_components"),
                                      ({"n_components": 2.5}, "n_components"), ({"max_iter": 0}, "max_iter"),
                                      ({"tol": -1e-3}, "tol"), ({"reg_covar": -1.0}, "reg_covar")])
def test_out_of_range_arguments_raise_before_launching(kw, match):
    with pytest.raises(ValueError, match=match):
        mixture.GaussianMixture(**kw)


def test_too_few_samples_raise_before_launching():
    with pytest.raises(ValueError, match="Expected n_samples >= n_components but got n_components = 5, n_samples = 3"):
        mixture.GaussianMixture(5).fit(np.zeros((3, 2)))
    with pytest.raises(ValueError, match="minimum of 2 is required"):
        mixture.GaussianMixture(1).fit(np.zeros((1, 2)))


def test_new_entry_points_are_declared_and_bound():
    names = {"tip_gmm_scatter_chunks", "tip_gmm_work_bytes", "tip_gmm_quad", "tip_gmm_resp", "tip_gmm_moments",
             "tip_gmm_scatter"}
    assert names <= set(_lib.symbols())
    lib = _lib.load()
    for name in names:
        assert hasattr(lib, name)


def test_scatter_chunks_follow_the_scratch_cap():
    lib = _lib.load()
    per_chunk = lambda d, k: k * ((d + 63) // 64) * ((d + 63) // 64 + 1) // 2 * 64 * 64 * 8
    for n, d, k in [(6000, 2048, 3), (100003, 2048, 1), (100003, 2048, 64)]:
        c = lib.tip_gmm_scatter_chunks(n, d, k, 1000)
        assert c >= 1 and (c == 1 or c * per_chunk(d, k) <= 256 << 20)
        assert c == 1 or (c + 1) * per_chunk(d, k) > 256 << 20 or c == n // 256
    assert lib.tip_gmm_scatter_chunks(6000, 2048, 3, 1) == 1
    assert lib.tip_gmm_scatter_chunks(6000, 128, 3, 0) > 1           # few output tiles: split over rows
    assert lib.tip_gmm_work_bytes(10, 0, 3, 0) == -1 and lib.tip_gmm_work_bytes(10, 4, 65, 0) == -1
