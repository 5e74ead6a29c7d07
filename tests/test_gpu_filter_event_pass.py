"""The resident DSA filter's one-pass tile epilogue under event storms, at 192-row query tiles.

Per row and tile the consumers reduce the four 32-column chunks at once, move the row's running minimum and threshold
once, to the tile's minimum, and record every chunk inside that end-of-tile threshold with the mask of its columns
inside it (DESIGN.md §4).  These inputs make many chunks records: training rows ordered so that each query's distance
falls along the scan, exact ties on both sides of a chunk and of a tile boundary, minima in a tile's last chunk and
duplicated rows.  For both stages and both input dtypes each case checks

* `dist_a`, `dist_b`, the winner and `dsa` bit for bit against the C oracle (eager launch, capture, replay);
* that no candidate list overflows;
* that every column a candidate mask admits is inside the window of its own chunk's minimum: with the accumulator
  modelled on the host (bf16 operands, exact products, error +-g) and the kernel's threshold formula taken at its
  widest, an admitted row's value is at most T(the chunk's smallest value).  A mask built against a threshold from
  before the chunk's own minimum arrived (an earlier, wider one) admits rows the descending case puts outside it."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle.filter_oracle import _bf16
from oracle.filter_oracle import threshold_hi as _thr_hi

pytestmark = pytest.mark.gpu

CLS, PER = 4, 1024          # class sizes are multiples of the 128-row train tile, so chunk / tile edges are global


def _descending(rng, dtype):
    # every class around one centre, its rows' radii falling along the class: each query's distance falls with the
    # scan of its own class (stage 1) and of each other class (stage 2), so nearly every chunk improves the minimum
    d = 128
    centre = rng.normal(size=d) * 3.0
    dirs = rng.normal(size=(CLS * PER, d))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    radius = np.tile(np.linspace(20.0, 0.5, PER), CLS) * (1 + 0.02 * rng.random(CLS * PER))
    xtr = (centre + dirs * radius[:, None]).astype(dtype)
    ytr = np.repeat(np.arange(CLS), PER)
    m = 500
    xte = (centre + rng.normal(size=(m, d)) * 0.01).astype(dtype)
    pte = rng.integers(0, CLS, size=m)
    return xtr, ytr, xte, pte


def _placed(rng, dtype):
    # ties across chunk (32) and tile (128) edges, minima in a tile's last chunk, duplicated rows
    d = 128
    centres = rng.normal(size=(CLS, d)) * 4.0
    ytr = np.repeat(np.arange(CLS), PER)
    xtr = (centres[ytr] + rng.normal(size=(CLS * PER, d))).astype(dtype)
    targets = []
    for c in range(CLS):
        o = c * PER
        for edge in (32, 160, 416, 128, 512, 896):         # chunk edges inside a tile, then tile edges
            xtr[o + edge] = xtr[o + edge - 1]
            targets.append(o + edge - 1)
        for j in (100, 127, 355, 1023):                    # inside the last chunk of their tile
            targets.append(o + j)
        for j in (7, 300, 700):                            # one row, four copies in four tiles
            for k in (1, 2, 3):
                xtr[o + (j + 256 * k) % PER] = xtr[o + j]
            targets.append(o + j)
    targets = np.repeat(np.array(targets), 12)
    xte = (xtr[targets] + rng.normal(size=(len(targets), d)) * 1e-3).astype(dtype)
    pte = ytr[targets]
    filler = rng.integers(0, CLS, size=120)                # ordinary queries, so query tiles mix both kinds
    xte = np.concatenate([xte, (centres[filler] + rng.normal(size=(120, d))).astype(dtype)])
    pte = np.concatenate([pte, filler])
    return xtr, ytr, xte, pte


def _check_bits(xtr, ytr, xte, pte):
    from simple_tip_b200.core.surprise import DSA

    want = c_oracle.dsa(xtr, ytr, xte, pte)
    sa = DSA(xtr, ytr)
    for _ in range(3):          # eager launch, graph capture, graph replay
        got = sa(xte, pte)
        assert np.array_equal(got, want["dsa"])
        assert np.array_equal(sa.last_winner_index, want["idx_a"])
        assert np.array_equal(sa.last_dist_a, want["dist_a"]) and np.array_equal(sa.last_dist_b, want["dist_b"])
    return sa


def _check_masks(eng, q, qcls, mode):
    """Runs one search of `mode` and checks its candidate lists; returns how many in-range columns of the candidate
    chunks lie outside their chunk's window (the columns an exact mask must drop)."""
    import torch

    from simple_tip_b200 import _lib

    q_off = np.searchsorted(qcls, np.arange(CLS + 1)).astype(np.int64)
    eng.search(q, torch.from_numpy(qcls.astype(np.int32)).to(eng.dev), q_off, mode)
    cnt, idx = (t.cpu().numpy() for t in eng.last_cand_cnt_by_mode[mode])
    assert cnt.max() <= eng.cap, "a candidate list overflowed"
    assert cnt.min() >= 1
    mu = eng.center.cpu().numpy().astype(np.float64)
    t = eng.t.cpu().numpy()
    x = q.cpu().numpy()
    yb = _bf16((t.astype(np.float64) - mu) if t.dtype == np.float64 else (t - mu.astype(np.float32)))
    xt = (x.astype(np.float64) - mu).astype(np.float32) if x.dtype == np.float64 else x - mu.astype(np.float32)
    xb = _bf16(xt)
    ysq = np.sum(yb.astype(np.float64) ** 2, axis=1)
    k16 = (((eng.d + 15) // 16) * 16 + 16) // 16
    gamma = (k16 * 16 + 16) * 2.0 ** -23
    off = eng.class_off
    outside = 0
    for i in range(x.shape[0]):
        nx = float(np.sum(xb[i].astype(np.float64) ** 2))
        errq = float(np.sqrt(np.sum((xt[i].astype(np.float64) - xb[i]) ** 2)))
        r = np.sqrt(nx) * (1 + 1e-6) + eng.rmax
        e2 = 2.0 * (errq + eng.errmax + 1.2e-7 * r) * 1.001
        g = gamma * r * r * 1.001
        lo, hi = off[qcls[i]], off[qcls[i] + 1]
        for col, mask in idx[i, :cnt[i]]:
            cols = col + np.arange(32)
            ok = cols < eng.n
            ok &= ((cols >= lo) & (cols < hi)) if mode == _lib.RANGE_SAME_CLASS else ((cols < lo) | (cols >= hi))
            bits = ((np.uint32(mask) >> np.arange(32, dtype=np.uint32)) & 1).astype(bool)
            assert bits.any() and not (bits & ~ok).any(), (i, col, hex(mask & 0xFFFFFFFF))
            acc = ysq[cols[ok]] - 2.0 * (yb[cols[ok]].astype(np.float64) @ xb[i].astype(np.float64))
            thr = _thr_hi(max(acc.min() + g + nx, 0.0) * (1 + 2.0 ** -22), nx, e2, g)
            adm = bits[ok]
            assert np.all(acc[adm] - g <= thr), (i, col, float((acc[adm] - g).max()), thr)
            outside += int(np.sum(acc - g > thr))
    return outside


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("case", ["descending", "placed"])
def test_event_storm_bits_and_exact_masks(case, dtype):
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    rng = np.random.default_rng({"descending": 11, "placed": 12}[case])
    xtr, ytr, xte, pte = (_descending if case == "descending" else _placed)(rng, dtype)
    sa = _check_bits(xtr, ytr, xte, pte)
    eng = sa._engine              # training traces of the test's dtype: the engine computes in it
    assert (eng.row_tile, eng.col_tile) == (192, 128), "these cases are meant for the resident 192-row filter"
    order = np.argsort(pte, kind="stable")
    qcls = pte[order]
    x = E.to_device(xte[order], eng.dev)
    assert x.dtype == eng.t.dtype
    outside = _check_masks(eng, x, qcls, _lib.RANGE_SAME_CLASS)
    w = eng.gather(eng.search(x, torch.from_numpy(qcls.astype(np.int32)).to(eng.dev),
                              np.searchsorted(qcls, np.arange(CLS + 1)).astype(np.int64), _lib.RANGE_SAME_CLASS)[1])
    outside += _check_masks(eng, w, qcls, _lib.RANGE_OTHER_CLASSES)
    if case == "descending":
        # teeth: the candidate chunks do hold in-range columns outside their window, which the masks left out
        assert outside > 0
