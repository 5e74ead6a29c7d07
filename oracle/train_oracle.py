"""NumPy references of the training kernels of simple_tip_b200/csrc/train.cu (TEST INFRASTRUCTURE ONLY).

  xent_reference(z, y)     the softmax cross-entropy head in float64, row by row, with no cancellation of its own
  xent_bounds(z, y)        what tip_softmax_xent's float32 operation order supports against xent_reference
  adam_restatement(...)    tip_keras_adam's float32 operation order (include/b200tip.h), bit for bit
  keras_adam_f64(...)      Keras' Adam in TF's ApplyAdam form, in float64
  torch_adam_f64(...)      the same with torch's epsilon on sqrt(v_hat); only used to show the Adam bound is sharp
  keras_adam_bound(...)    what the float32 order supports against keras_adam_f64
  gather_reference(...)    tip_stack_gather as NumPy fancy indexing, then astype(float32)

The bounds are derived from the kernels' operation order below, with u = 2^-24 (half an ulp of 1 in float32), not
fitted to a run.  Inputs are NumPy arrays; nothing in the product package imports this module.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Sequence, Tuple

import numpy as np

F = np.float32
U = 2.0 ** -24
# an absolute floor for the float32 underflow: a row's loss sums at most 32 lanes, each of whose terms carries a few
# subnormal ulps (2^-149) when o or y * (-log p) underflows; 32 * 2^-126 is far above that and far below any loss
# the tests look at
XENT_LOSS_FLOOR = 32 * 2.0 ** -126
# dz: expf at 2 subnormal ulps, then the division by s, the subtraction of y and the division by the row count
XENT_DZ_FLOOR = 8 * 2.0 ** -149


class Xent(NamedTuple):
    nlp: np.ndarray          # [R, C] -log p_c (+inf where z_c = -inf)
    loss: np.ndarray         # [R]    sum_c y_c * (-log p_c), terms with y_c = 0 left out
    dz: np.ndarray           # [R, C] softmax - y (not divided by the row count)
    argmax_z: np.ndarray     # [R]    first index of the max of z
    argmax_y: np.ndarray     # [R]    first index of the max of y
    p: np.ndarray            # [R, C] softmax
    d: np.ndarray            # [R, C] max(z) - z_c >= 0


def xent_reference(z: np.ndarray, y: np.ndarray) -> Xent:
    """The softmax cross-entropy of float32 logits z [R, C] against targets y [R, C] in float64, row by row.

    With d_c = max(z) - z_c, n_top lanes at the max and rest = sum of exp(-d_c) over the lanes below it:
    -log p_c = d_c + log1p((n_top - 1) + rest) (log-sum-exp), and 1 - p_c = sum_{c' != c} p_c' = ((n_top - 1) +
    rest) / s at a lane of the max and (n_top + (rest - e_c)) / s below it (>= 1 / s: no cancellation), s = n_top +
    rest.  dz is -(1 - p_c) where y_c = 1 and p_c - y_c elsewhere.  The max of each row must be finite."""
    z = np.asarray(z, dtype=F).astype(np.float64)
    y = np.asarray(y, dtype=F).astype(np.float64)
    mx = z.max(axis=1, keepdims=True)
    assert np.all(np.isfinite(mx)), "every row needs a finite max"
    d = mx - z
    e = np.exp(-d)
    top = d == 0
    n_top = top.sum(axis=1, keepdims=True).astype(np.float64)
    rest = np.where(top, 0.0, e).sum(axis=1, keepdims=True)
    s = n_top + rest
    nlp = d + np.log1p((n_top - 1) + rest)
    p = e / s
    others = np.where(top, (n_top - 1) + rest, n_top + (rest - e))
    dz = np.where(y == 1, -others / s, p - y)
    with np.errstate(invalid="ignore"):
        loss = np.where(y != 0, y * nlp, 0.0).sum(axis=1)
    return Xent(nlp, loss, dz, np.argmax(z, axis=1), np.argmax(y, axis=1), p, d)


def xent_bounds(z: np.ndarray, y: np.ndarray, ref: Optional[Xent] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(loss [R], dz [R, C]): bounds on |kernel - xent_reference| of each row's loss and of each dz entry before
    the division by the row count.

    The kernel's order per row: t_c = z_c - mx (rounded: relative error u, so exp(t_c) is off by up to d_c * u),
    e_c = expf(t_c) (2 ulp = 4u), s = a 5-level tree sum of the e_c, o_k = the same tree with lane k zeroed,
    -log p = log1pf(o_k) at a lane of the max, (mx - z_c) + logf(s) below it (logf, log1pf: 1 ulp = 2u; 4u
    assumed), y_c * (-log p) rounded once, the lanes summed in a 5-level tree, the row sums in double.  With D = the
    p-weighted mean of d over the lanes below the max (0 if none carries weight), s and every o_k are within
    (9 + D) u relative.  So:
      * a lane of the max: |log1pf(o) - log1p(O)| <= 2u l + (9 + D) u O / (1 + O) <= (11 + D) u l, since
        O / (1 + O) <= log1p(O);
      * a lane below it: u d + (9 + D) u + 2u L + u (d + L) <= (17 + 1.5 D) u l, since l = d + L >= log 2 there;
      * the product by y and the tree of positive terms add 6u: per row |loss - loss*| <= (23 + 1.5 D) u
        sum_c y_c l_c.  The bound is (32 + 2 D) u sum_c y_c l_c + XENT_LOSS_FLOOR.
    dz (its magnitude mag = |p - y| where y_c = 1, else p + y):
      * y_c = 1: -o / s, (9 + D) u for o and s each, u for the division and u for the one by the row count:
        (20 + 2 D) u |p - 1|;
      * else e / s - y: p (4 + d_c + 9 + D + 1) u from e, s and the division, u (p + y) for the subtraction and the
        division by the row count: (16 + D) u (p + y) + u p d_c.
      The bound is u ((32 + 2 D) mag + 2 p d) + XENT_DZ_FLOOR.
    Where the reference loss is +inf (a -inf logit under a nonzero target) the kernel must give +inf too."""
    ref = xent_reference(z, y) if ref is None else ref
    y = np.asarray(y, dtype=F).astype(np.float64)
    below = ref.d > 0
    with np.errstate(invalid="ignore"):
        pd = np.where(ref.p > 0, ref.p * ref.d, 0.0)
        nl = np.where(y != 0, np.abs(y) * ref.nlp, 0.0).sum(axis=1)
    wsum = np.where(below, ref.p, 0.0).sum(axis=1, keepdims=True)
    D = np.where(wsum > 0, pd.sum(axis=1, keepdims=True) / np.where(wsum > 0, wsum, 1.0), 0.0)
    k = 32.0 + 2.0 * D
    loss = U * k[:, 0] * nl + XENT_LOSS_FLOOR
    mag = np.where(y == 1, np.abs(ref.dz), ref.p + np.abs(y))
    dz = U * (k * mag + 2.0 * pd) + XENT_DZ_FLOOR
    return loss, dz


def xent_bank(rng: np.random.Generator, n: int, classes: int, inf_targets: bool = True):
    """(z, y) float32 [n, classes]: rows at the head's edges, row i of logit kind i % 8 and target kind (i // 8) % 6.
    Logits: normal with sigma 1e-3, 4 and 30; the true class leading the others by 5..40; all equal; ties for the
    max; -inf entries (under a nonzero target in every third such row when inf_targets, else only under zero
    targets); a spread of +-1e-3..1e30.  Targets: one-hot, label-smoothed (0.1), Dirichlet, two ones, all zero,
    and a tie of two halves.  +-3e38 is left out: there mx - z overflows in float32 but not in float64."""
    c = classes
    z = np.empty((n, c), dtype=np.float64)
    y = np.zeros((n, c), dtype=np.float64)
    for i in range(n):
        zk, yk = i % 8, (i // 8) % 6
        label = int(rng.integers(c))
        other = (label + 1 + int(rng.integers(max(c - 1, 1)))) % c
        if yk == 0 or (c == 1 and yk in (3, 5)):
            y[i, label] = 1.0
        elif yk == 1:
            y[i] = 0.1 / c
            y[i, label] += 0.9
        elif yk == 2:
            y[i] = rng.dirichlet(np.ones(c))
        elif yk == 3:
            y[i, [label, other]] = 1.0
        elif yk == 5:
            y[i, [label, other]] = 0.5
        if zk == 0:
            z[i] = rng.normal(size=c) * 1e-3
        elif zk == 1 or (c == 1 and zk in (3, 5, 6)):
            z[i] = rng.normal(size=c) * 4
        elif zk == 2:
            z[i] = rng.normal(size=c) * 30
        elif zk == 3:
            z[i] = rng.normal(size=c)
            z[i, label] = np.delete(z[i], label).max() + rng.uniform(5, 40)
        elif zk == 4:
            z[i] = rng.normal() * 10
        elif zk == 5:
            z[i] = np.round(rng.normal(size=c) * 2)
            z[i, rng.choice(c, size=min(c, int(rng.integers(2, 4))), replace=False)] = z[i].max()
        elif zk == 6:
            z[i] = rng.normal(size=c) * 4
            lanes = np.arange(c) if inf_targets else np.flatnonzero(y[i] == 0)
            lanes = set(lanes[rng.random(lanes.size) < 0.5].tolist())
            if inf_targets and i % 3 == 0:
                lanes.add(label)
            lanes.discard(other)                          # the max stays finite
            z[i, sorted(lanes)] = -np.inf
        else:
            z[i] = rng.choice([-1.0, 1.0], size=c) * 10.0 ** rng.uniform(-3, 30, size=c)
    return z.astype(F), y.astype(F)


def adam_restatement(p: np.ndarray, grads: Sequence[np.ndarray], t0: int = 0, lr=1e-3, beta1=0.9, beta2=0.999,
                     epsilon=1e-7, m: Optional[np.ndarray] = None, v: Optional[np.ndarray] = None):
    """tip_keras_adam's order (include/b200tip.h) over steps t0 + 1 .. t0 + len(grads): every operation in float32,
    rounded once; beta^t in float64, rounded once.  Returns (p, m, v) as float32; m and v start at 0 unless given.
    Overflow and NaN propagate as in IEEE float32 (NumPy does not flush subnormals)."""
    lr, b1, b2, eps, one = F(lr), F(beta1), F(beta2), F(epsilon), F(1)
    p = np.array(p, dtype=F)
    m = np.zeros_like(p) if m is None else np.array(m, dtype=F)
    v = np.zeros_like(p) if v is None else np.array(v, dtype=F)
    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        for t, g in enumerate(grads, start=t0 + 1):
            g = np.asarray(g, dtype=F)
            b1t, b2t = F(np.float64(b1) ** t), F(np.float64(b2) ** t)
            lr_t = F(lr * F(F(np.sqrt(F(one - b2t))) / F(one - b1t)))
            m = F(b1 * m) + F(F(one - b1) * g)
            v = F(b2 * v) + F(F(one - b2) * F(g * g))
            p = p - F(lr_t * m) / F(np.sqrt(v) + eps)
    return p, m, v


def _f64(*hyper):
    """Keras keeps its hyperparameters as float32 variables: the float64 references start from those values."""
    return [np.float64(F(h)) for h in hyper]


def keras_adam_f64(p, grads, t0: int = 0, lr=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-7, m=None, v=None):
    """Keras' Adam in TF's ApplyAdam form, in float64: alpha = lr sqrt(1 - b2^t) / (1 - b1^t), m += (g - m)(1 - b1),
    v += (g^2 - v)(1 - b2), p -= alpha m / (sqrt(v) + eps).  Returns float64 (p, m, v)."""
    lr, b1, b2, eps = _f64(lr, beta1, beta2, epsilon)
    p = np.array(p, dtype=np.float64)
    m = np.zeros_like(p) if m is None else np.array(m, dtype=np.float64)
    v = np.zeros_like(p) if v is None else np.array(v, dtype=np.float64)
    for t, g in enumerate(grads, start=t0 + 1):
        g = np.asarray(g, dtype=np.float64)
        alpha = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        m = m + (g - m) * (1 - b1)
        v = v + (g * g - v) * (1 - b2)
        p = p - alpha * m / (np.sqrt(v) + eps)
    return p, m, v


def torch_adam_f64(p, grads, t0: int = 0, lr=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-7, m=None, v=None):
    """torch.optim.Adam's form in float64: p -= lr m_hat / (sqrt(v_hat) + eps), m_hat = m / (1 - b1^t),
    v_hat = v / (1 - b2^t).  It differs from Keras' by where epsilon sits."""
    lr, b1, b2, eps = _f64(lr, beta1, beta2, epsilon)
    p = np.array(p, dtype=np.float64)
    m = np.zeros_like(p) if m is None else np.array(m, dtype=np.float64)
    v = np.zeros_like(p) if v is None else np.array(v, dtype=np.float64)
    for t, g in enumerate(grads, start=t0 + 1):
        g = np.asarray(g, dtype=np.float64)
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        p = p - lr * (m / (1 - b1 ** t)) / (np.sqrt(v / (1 - b2 ** t)) + eps)
    return p, m, v


def keras_adam_bound(p, grads, t0: int = 0, lr=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-7, m=None, v=None):
    """(p, m, v): bounds on |float32 order - keras_adam_f64| after len(grads) steps, for finite, normal gradients
    (no subnormal or overflowing intermediate), from error recurrences run beside the float64 Adam:
      * lr_t: b2t = fl32(b2^t) is off by u b2^t, which 1 - b2t (exact for b2t >= 1/2) turns into u b2^t / (1 - b2^t)
        relative and the square root halves; likewise u b1^t / (1 - b1^t) from 1 - b1t; the square root, the
        division, the product by lr and a subtraction below 1/2 add up to 4u: r_a = u (b2^t / (2 (1 - b2^t)) +
        b1^t / (1 - b1^t) + 4);
      * m: E_m <- b1 E_m + u (b1 |m_prev| + (1 - b1) |g| + |m|) (two products and a sum, each rounded once);
      * v (positive terms): E_v <- b2 E_v + u (b2 v_prev + 2 (1 - b2) g^2 + v);
      * the denominator: E_den = sqrt(v) E_v / (2 v) + 2u (sqrt(v) + eps) (sqrt and the sum with eps, rounded);
      * the step A = alpha |m| / den: E_A = A (r_a + E_den / den + 2u) + alpha E_m / den (the product by lr_t and
        the division, rounded once each);
      * p: E_p <- E_p + E_A + u |p| (the subtraction).
    The first-order recurrences use the float64 run's values for the float32 ones; the bounds returned are twice the
    recurrences, which covers the second-order terms by a wide margin."""
    lr, b1, b2, eps = _f64(lr, beta1, beta2, epsilon)
    p = np.array(p, dtype=np.float64)
    m = np.zeros_like(p) if m is None else np.array(m, dtype=np.float64)
    v = np.zeros_like(p) if v is None else np.array(v, dtype=np.float64)
    ep, em, ev = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
    for t, g in enumerate(grads, start=t0 + 1):
        g = np.asarray(g, dtype=np.float64)
        b1t, b2t = b1 ** t, b2 ** t
        alpha = lr * np.sqrt(1 - b2t) / (1 - b1t)
        r_a = U * (b2t / (2 * (1 - b2t)) + b1t / (1 - b1t) + 4)
        m_new = m + (g - m) * (1 - b1)
        v_new = v + (g * g - v) * (1 - b2)
        em = b1 * em + U * (b1 * np.abs(m) + (1 - b1) * np.abs(g) + np.abs(m_new))
        ev = b2 * ev + U * (b2 * v + 2 * (1 - b2) * g * g + v_new)
        m, v = m_new, v_new
        root = np.sqrt(v)
        den = root + eps
        e_den = np.where(v > 0, root * ev / (2 * np.where(v > 0, v, 1.0)), 0.0) + 2 * U * den
        step = alpha * np.abs(m) / den
        p = p - alpha * m / den
        ep = ep + step * (r_a + e_den / den + 2 * U) + alpha * em / den + U * np.abs(p)
    return 2 * ep, 2 * em, 2 * ev


def gather_reference(pool: np.ndarray, rows: np.ndarray, perm: np.ndarray, start: int, b: int,
                     interleaved: bool) -> np.ndarray:
    """tip_stack_gather: row j < b of model m is pool[rows[m, perm[m, start + j]]]; a float64 pool is rounded to
    float32 to nearest (ties to even, beyond FLT_MAX to inf).  interleaved: [M, b, H, W, C] -> [b, H, W, M * C]."""
    idx = np.take_along_axis(np.asarray(rows), np.asarray(perm)[:, start:start + b], axis=1)
    got = np.asarray(pool)[idx]
    if got.dtype == np.float64:
        with np.errstate(over="ignore"):
            got = got.astype(F)
    if interleaved:
        m, b_, h, w, c = got.shape
        got = got.transpose(1, 2, 3, 0, 4).reshape(b_, h, w, m * c)
    return np.ascontiguousarray(got)
