"""The resident DSA filter builds a chunk's column mask only where a row of the warp has an event in that chunk.

Two cases at 192-row query tiles, both stages and both input dtypes:

* every chunk an event: each class's training rows start with one 128-row tile of identical rows, so on that tile
  every query row of a warp has its minimum in all four chunks, in both row halves at once;
* exactly one: one query per class (row 0 of its query tile, so one row half of one warp), training rows ordered by
  growing distance and one near copy of the query in chunk 2 of a later tile, so on that tile exactly one (row half,
  chunk) of the warp has an event.

Each checks `dist_a`, `dist_b`, the winner and `dsa` bit for bit against the C oracle (eager launch, capture, replay)
and that every candidate mask admits exactly columns inside their chunk's window."""
import numpy as np
import pytest

from tests.test_gpu_filter_event_pass import CLS, PER, _check_bits, _check_masks

pytestmark = pytest.mark.gpu


def _all_chunks(rng, dtype):
    d = 128
    centres = rng.normal(size=(CLS, d)) * 4.0
    ytr = np.repeat(np.arange(CLS), PER)
    xtr = centres[ytr] + rng.normal(size=(CLS * PER, d))
    for c in range(CLS):
        xtr[c * PER:c * PER + 128] = centres[c] + 0.05 * rng.normal(size=d)
    m = 400
    pte = rng.integers(0, CLS, size=m)
    xte = centres[pte] + rng.normal(size=(m, d)) * 0.01
    return xtr.astype(dtype), ytr, xte.astype(dtype), pte


def _one_chunk(rng, dtype):
    d = 128
    centres = rng.normal(size=(CLS, d)) * 3.0
    ytr = np.repeat(np.arange(CLS), PER)
    dirs = rng.normal(size=(CLS * PER, d))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    radius = np.tile(np.linspace(5.0, 40.0, PER), CLS)
    xtr = centres[ytr] + dirs * radius[:, None]
    pte = np.arange(CLS)
    xte = centres.copy()
    for c in range(CLS):
        xtr[c * PER + 5 * 128 + 2 * 32 + 7] = xte[c] + 1e-3 * rng.normal(size=d)
    return xtr.astype(dtype), ytr, xte.astype(dtype), pte


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("case", ["all_chunks", "one_chunk"])
def test_event_masks_bits_and_exact(case, dtype):
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    rng = np.random.default_rng({"all_chunks": 21, "one_chunk": 22}[case])
    xtr, ytr, xte, pte = (_all_chunks if case == "all_chunks" else _one_chunk)(rng, dtype)
    sa = _check_bits(xtr, ytr, xte, pte)
    eng = sa._engine
    assert (eng.row_tile, eng.col_tile) == (192, 128), "these cases are meant for the resident 192-row filter"
    order = np.argsort(pte, kind="stable")
    qcls = pte[order]
    x = E.to_device(xte[order], eng.dev)
    _check_masks(eng, x, qcls, _lib.RANGE_SAME_CLASS)
    q_off = np.searchsorted(qcls, np.arange(CLS + 1)).astype(np.int64)
    w = eng.gather(eng.search(x, torch.from_numpy(qcls.astype(np.int32)).to(eng.dev), q_off, _lib.RANGE_SAME_CLASS)[1])
    _check_masks(eng, w, qcls, _lib.RANGE_OTHER_CLASSES)
