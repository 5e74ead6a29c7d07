"""CPU tests of the device EmpiricalCovariance backend's host side: backend selection, the errors raised before any
launch, and the export table of the new entry point."""
import numpy as np
import pytest

from simple_tip_b200 import _lib
from simple_tip_b200.core import covariance
from simple_tip_b200.core.surprise import MDSA, MultiModalSA


def _rows():
    return np.random.RandomState(42).random((60, 4))


def test_sklearn_backend_stays_the_default(monkeypatch):
    monkeypatch.delenv("B200TIP_COV", raising=False)
    m = MDSA(_rows())
    assert m.backend == "sklearn"
    assert type(m.covariance_matrix).__module__.startswith("sklearn")


def test_unknown_backend_is_rejected(monkeypatch):
    with pytest.raises(ValueError, match="backend"):
        MDSA(_rows(), backend="cpu")
    monkeypatch.setenv("B200TIP_COV", "cuda")
    with pytest.raises(ValueError, match="backend"):
        MDSA(_rows())


def test_device_backend_without_a_gpu_fails_loudly(monkeypatch):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        MDSA(_rows(), backend="device")
    monkeypatch.setenv("B200TIP_COV", "device")
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        MultiModalSA.build_by_class(_rows(), np.arange(60) % 2, lambda x, y: MDSA(x))
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        covariance.EmpiricalCovariance().fit(_rows())


@pytest.mark.parametrize("shape,match", [((0, 3), r"Found array with 0 sample\(s\) \(shape=\(0, 3\)\) while a minimum "
                                                  r"of 1 is required by EmpiricalCovariance"),
                                         ((3, 0), r"Found array with 0 feature\(s\) \(shape=\(3, 0\)\)"),
                                         ((5,), "2-dimensional"), ((2, 3, 4), "2-dimensional")])
def test_empty_or_malformed_input_raises_before_launching(shape, match):
    with pytest.raises(ValueError, match=match):
        covariance.EmpiricalCovariance().fit(np.zeros(shape))


def test_the_same_empty_input_is_what_sklearn_rejects():
    from sklearn.covariance import EmpiricalCovariance

    for shape in ((0, 3), (3, 0)):
        with pytest.raises(ValueError, match="Found array with 0"):
            EmpiricalCovariance().fit(np.zeros(shape))


def test_unfitted_estimator_raises():
    with pytest.raises(RuntimeError, match="not fitted"):
        covariance.EmpiricalCovariance().get_precision()


def test_new_entry_point_is_declared_and_bound():
    assert "tip_cov_location" in set(_lib.symbols())
    assert hasattr(_lib.load(), "tip_cov_location")
