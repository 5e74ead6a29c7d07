"""The closed form of the surprise-coverage CAM order (oracle/sc_oracle.py) against the greedy loop on the dense
profile (np_oracle.cam_oracle), and the threshold check that decides between the two (CPU only)."""
import numpy as np
import pytest

from oracle import np_oracle, sc_oracle
from simple_tip_b200.core.prioritizers import thresholds_one_hot
from simple_tip_b200.core.surprise import SurpriseCoverageMapper


def _edge_values(t: np.ndarray, dtype) -> np.ndarray:
    """Every finite threshold, one ulp either side of it, in `dtype`."""
    t = t[np.isfinite(t)]
    v = np.concatenate([t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)]).astype(dtype)
    return np.concatenate([v, np.nextafter(v, np.array(-np.inf, dtype)), np.nextafter(v, np.array(np.inf, dtype))])


def _cases():
    rng = np.random.default_rng(0)
    for dtype in (np.float32, np.float64):
        for sections in (1, 2, 1000):
            for overflow in (False, True):
                rep = rng.choice(rng.random(40) * 3.0, size=300).astype(dtype)                   # repeated values
                yield f"repeated-{dtype.__name__}-{sections}-{overflow}", rep, sections, overflow
                t = SurpriseCoverageMapper(sections, 2.5, overflow).thresholds
                edges = rng.permutation(_edge_values(t, dtype)[:3000])
                yield f"edges-{dtype.__name__}-{sections}-{overflow}", edges, sections, overflow
                nan = rng.random(200).astype(dtype)
                nan[rng.integers(0, 200, 30)] = np.nan
                yield f"nan-{dtype.__name__}-{sections}-{overflow}", nan, sections, overflow


CASES = list(_cases())


@pytest.mark.parametrize("name,values,sections,overflow", CASES, ids=[c[0] for c in CASES])
def test_closed_form_equals_the_greedy_loop(name, values, sections, overflow):
    ub = np.max(values) if not np.isnan(values).any() else 2.5
    mapper = SurpriseCoverageMapper(sections, ub, overflow)
    assert thresholds_one_hot(mapper.thresholds)
    want = np_oracle.cam_oracle(values, mapper.get_coverage_profile(values))
    assert np.array_equal(sc_oracle.sc_cam_oracle(values, mapper.thresholds), want)


def test_the_maximum_lies_outside_the_last_half_open_bucket():
    v = np.array([0.0, 0.5, 1.0, 1.0, 0.25])
    mapper = SurpriseCoverageMapper(4, np.max(v))
    assert sc_oracle.sc_buckets(v, mapper.thresholds).tolist() == [0, 2, -1, -1, 1]
    assert mapper.get_coverage_profile(v)[2].sum() == 0
    assert np.array_equal(sc_oracle.sc_cam_oracle(v, mapper.thresholds),
                          np_oracle.cam_oracle(v, mapper.get_coverage_profile(v)))


def test_golden_surprise_coverage_case(golden):
    s = golden("siblings_reference.npz")
    v = s["sc.values"]
    mapper = SurpriseCoverageMapper(1000, np.max(v))
    assert thresholds_one_hot(mapper.thresholds)
    assert np.array_equal(sc_oracle.sc_cam_oracle(v, mapper.thresholds), s["sc.cam"])


@pytest.mark.parametrize("overflow", [False, True])
@pytest.mark.parametrize("ub,one_hot", [(0.0, True), (1e-320, True), (1.0, True), (3.7e5, True), (1e300, True),
                                        (-1.0, False), (np.nan, False), (np.inf, False)])
def test_threshold_check(ub, one_hot, overflow):
    with np.errstate(invalid="ignore"):
        mapper = SurpriseCoverageMapper(1000, ub, overflow)
        assert thresholds_one_hot(mapper.thresholds) == one_hot
        if one_hot:
            finite = ub if np.isfinite(ub) else 1.0
            v = np.concatenate([_edge_values(mapper.thresholds, np.float64), [finite, -finite, np.nan, np.inf]])
            prof = mapper.get_coverage_profile(v)
            assert prof.sum(axis=1).max() <= 1
            assert np.array_equal(sc_oracle.sc_cam_oracle(v, mapper.thresholds), np_oracle.cam_oracle(v, prof))


def test_overflow_bucket_with_a_negative_bound_still_covers():
    """The dense path is not empty in every failing case: [t[-2], inf) of the overflow bucket still holds values."""
    with np.errstate(invalid="ignore"):
        mapper = SurpriseCoverageMapper(10, -1.0, overflow_bucket=True)
    assert mapper.get_coverage_profile(np.array([5.0, -0.5])).any()
