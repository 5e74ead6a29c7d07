"""CPU checks of the uncertainty-quantifier oracle (oracle/quantifier_oracle.py): hand-computed answers, two
independent restatements (scipy.stats.entropy, scipy.stats.mode), and the class-method surface of the product
classes, which needs no GPU."""
import numpy as np
import pytest
import scipy.stats

from oracle import quantifier_oracle as Q


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_known_answers(dt):
    p = np.array([[.5, .25, .25], [.5, .5, 0], [0, 0, 1], [.25, .5, .25]], dtype=dt)
    pred, ent = Q.softmax_entropy(p)
    assert ent.dtype == dt and ent[0] == 1.5 and ent[3] == 1.5
    assert ent[1] == 1.0                     # the 1e-20 in place of 0 adds 6.6e-19: below half an ulp of 1
    assert ent[2] == 0.0 or abs(ent[2]) < 1e-17
    assert np.array_equal(pred, [0, 0, 2, 1])
    pred, pc = Q.pcs(p)
    assert pc.dtype == dt and pc[0] == 0.25 and pc[1] == 0.0 and pc[2] == 1.0 and pc[3] == 0.25
    assert np.array_equal(pred, [0, 0, 2, 1])   # first index on ties
    pred, mx = Q.max_softmax(p)
    assert np.array_equal(mx, np.array([.5, .5, 1, .5], dtype=dt))
    assert p[1, 2] == 0                       # the input is not modified


def test_pcs_needs_two_classes():
    with pytest.raises(ValueError):
        Q.pcs(np.ones((3, 1)))


def test_variation_ratio_ties_with_four_samples():
    # votes per row (S = 4, C = 3): [0 1 1 0] -> tie 0/1, mode 0; [2 2 1 1] -> tie 1/2, mode 1; [2 0 1 2] -> mode 2;
    # [1 1 1 1] -> unanimous
    votes = np.array([[0, 1, 1, 0], [2, 2, 1, 1], [2, 0, 1, 2], [1, 1, 1, 1]])
    p = np.full(votes.shape + (3,), 0.1)
    np.put_along_axis(p, votes[..., None], 0.8, axis=2)
    pred, vr = Q.variation_ratio(p)
    assert np.array_equal(pred, [0, 1, 2, 1])
    assert vr.dtype == np.float64 and np.array_equal(vr, [0.5, 0.5, 0.5, 0.0])


def test_entropy_agrees_with_scipy_on_positive_rows():
    rng = np.random.default_rng(0)
    for c in (2, 10, 1000):
        p = rng.dirichlet(np.full(c, 0.3), size=200)
        p = np.maximum(p, 1e-300)
        _, ent = Q.softmax_entropy(p)
        want = scipy.stats.entropy(p, base=2, axis=1)        # normalises first; p sums to 1 within rounding
        np.testing.assert_allclose(ent, want, rtol=1e-12, atol=1e-12)
        _, ent32 = Q.softmax_entropy(p.astype(np.float32))
        np.testing.assert_allclose(ent32, want, rtol=2e-5, atol=2e-5)


def test_variation_ratio_tie_rule_is_scipy_mode():
    rng = np.random.default_rng(1)
    for s, c in ((4, 3), (7, 2), (200, 10), (5, 50)):
        p = rng.dirichlet(np.ones(c), size=(300, s))
        votes = np.argmax(p, axis=2)
        mode = scipy.stats.mode(votes, axis=1, keepdims=False)
        pred, vr = Q.variation_ratio(p)
        assert np.array_equal(pred, mode.mode)
        assert np.array_equal(vr, 1 - mode.count / s)


def test_pcs_counts_duplicates_like_a_sort():
    rng = np.random.default_rng(2)
    p = rng.integers(0, 4, size=(500, 6)).astype(np.float32) / 4       # many repeated values
    _, pc = Q.pcs(p)
    top = np.sort(p, axis=1)
    assert np.array_equal(pc, top[:, -1] - top[:, -2])
    assert np.all(pc[(p == p.max(axis=1, keepdims=True)).sum(axis=1) > 1] == 0)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_nan_rows_follow_numpy(dt):
    """The NaN rules of the contract: the first NaN is the prediction and the vote, and its row's values are NaN."""
    nan, inf = np.nan, np.inf
    p = np.array([[.2, nan, .7, nan], [nan, .1, .2, .3], [.1, .2, .3, nan], [inf, nan, .1, .2],
                  [nan, nan, nan, nan], [inf, .1, inf, .2], [-inf, -inf, -inf, -inf], [.1, .6, .6, .2]], dtype=dt)
    want_pred = [1, 0, 3, 1, 0, 0, 0, 1]
    with np.errstate(invalid="ignore"):
        for f in (Q.max_softmax, Q.pcs, Q.softmax_entropy):
            assert np.array_equal(f(p)[0], want_pred), f.__name__
        mx, pc, ent = Q.max_softmax(p)[1], Q.pcs(p)[1], Q.softmax_entropy(p)[1]
    assert np.all(np.isnan(mx[:5])) and mx[5] == inf and mx[6] == -inf and mx[7] == dt(.6)
    assert np.all(np.isnan(pc[:7])) and pc[7] == 0                  # inf - inf and -inf - -inf are NaN too
    assert np.all(np.isnan(ent[:5])) and np.isnan(ent[6]) and ent[5] == -inf
    votes = np.broadcast_to(p[:5, None, :], (5, 3, 4))             # three samples of the NaN rows
    assert np.array_equal(Q.vote_counts(votes).argmax(axis=1), want_pred[:5])
    pred, vr = Q.variation_ratio(votes)
    assert np.array_equal(pred, want_pred[:5]) and np.array_equal(vr, np.zeros(5))


def test_product_classes_have_the_uwiz_surface():
    from simple_tip_b200.core import quantifiers as P
    from simple_tip_b200.core.deepgini import DeepGini

    want = {P.MaxSoftmax: ("softmax", False, True), P.PredictionConfidenceScore: ("pcs", False, True),
            P.SoftmaxEntropy: ("softmax_entropy", False, False), P.VariationRatio: (None, True, False)}
    for cls, (alias, samples, conf) in want.items():
        assert issubclass(cls, DeepGini.__mro__[1])
        if alias is not None:
            assert cls.aliases()[0] == alias                  # the study names its result files after it
        assert cls.takes_samples() is samples and cls.is_confidence() is conf
        assert cls.problem_type() == DeepGini.problem_type()
        x = np.array([0.25, 0.5])
        assert np.array_equal(cls.cast_conf_or_unc(False, x), -x if conf else x)
        assert np.array_equal(cls.cast_conf_or_unc(None, x), x)
        assert np.array_equal(cls.cast_conf_or_unc(True, x), x if conf else -x)
        assert np.array_equal(Q.cast_conf_or_unc(conf, False, x), cls.cast_conf_or_unc(False, x))
