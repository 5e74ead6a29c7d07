"""The filter kernel's resident-query loop (pair_tc.cu): one wgmma commit group per K chunk, all committed before one
wait per tile, the tile-skipping epilogue of the nearest-neighbour mode, and the query tile kept resident across
consecutive work items of the same query tile.  Raw accumulators against the float64 product of the packed operands
for every K16 tail length, and DSA against the C oracle bit for bit over work lists of 1-, 2- and 3-tile items."""
import numpy as np
import pytest

from oracle import c_oracle, np_oracle

pytestmark = pytest.mark.gpu


# 1 segment: k16 = d/16 + 1, 3 segments: k16 = 3 d/16 + 1; the tail after the last full 4-step chunk is k16 % 4.
# Resident kernel: up to 5 K chunks (k16 <= 20), 5 of the 6 ring stages in flight before one wait.
@pytest.mark.parametrize("d,segments,tail", [(48, 1, 0), (64, 1, 1), (80, 1, 2), (96, 1, 3), (128, 1, 1),
                                             (288, 1, 3), (16, 3, 0), (64, 3, 1), (48, 3, 2), (32, 3, 3),
                                             (80, 3, 0), (96, 3, 3)])
@pytest.mark.parametrize("variant", [1, 2])
def test_probe_accumulators_every_tail(d, segments, tail, variant):
    import torch

    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E

    k16 = (segments * ((d + 15) // 16 * 16) + 16) // 16
    assert k16 % 4 == tail
    if variant == 2 and (k16 + 3) // 4 > 5:
        pytest.skip("packed row too wide for the resident-query kernel (5 K chunks)")
    lib = _lib.load()
    dev = E.require_cuda()
    rng = np.random.default_rng(100 * d + segments)
    q = torch.from_numpy(rng.normal(size=(256, d)).astype(np.float32)).to(dev)
    t = torch.from_numpy(rng.normal(size=(256, d)).astype(np.float32)).to(dev)
    center = torch.zeros(d, dtype=torch.float32, device=dev)
    pitch = int(lib.tip_pair_pitch(d, segments))
    qp = torch.empty((256, pitch), dtype=torch.bfloat16, device=dev)
    tp = torch.empty((256, pitch), dtype=torch.bfloat16, device=dev)
    qs, ts, qe = (torch.empty(256, dtype=torch.float32, device=dev) for _ in range(3))
    scale, coef = (-2.0, 1.0) if segments == 1 else (1.0, -0.5)
    _lib.check(lib.tip_pair_prep(E._p(q), _lib.TIP_F32, 256, d, E._p(center), _lib.ROLE_QUERY, segments, 1.0, 0.0,
                                 E._p(qp), E._p(qs), E._p(qe), E._stream()), "prep q")
    _lib.check(lib.tip_pair_prep(E._p(t), _lib.TIP_F32, 256, d, E._p(center), _lib.ROLE_TRAIN, segments, scale, coef,
                                 E._p(tp), E._p(ts), None, E._stream()), "prep t")
    out = torch.zeros((256, 256), dtype=torch.float32, device=dev)
    _lib.check(lib.tip_pair_probe(E._p(qp), 256, E._p(tp), 256, d, segments, pitch, variant, E._p(out), E._stream()),
               "probe")
    torch.cuda.synchronize()
    rows = int(lib.tip_kde_tile_rows())
    want = qp[:rows].to(torch.float64) @ tp.to(torch.float64).T
    mag = qp[:rows].to(torch.float64).abs() @ tp.to(torch.float64).abs().T
    err = (out[:rows].to(torch.float64) - want).abs()
    assert bool((err <= 4e-6 * mag + 1e-6).all()), float((err - 4e-6 * mag).max())


def _dsa_case(monkeypatch, pool_tiles, n_train, n_test, classes, d, seed, pool_frac=0.5):
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import DSA

    monkeypatch.setattr(E, "POOL_FRAC", pool_frac)
    monkeypatch.setattr(E, "POOL_TILES", pool_tiles)
    monkeypatch.setattr(E, "POOL_MIN_TILES", 0)
    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(n_train, n_test, d, classes, seed=seed)
    want = c_oracle.dsa(xtr, ytr, xte, pte)
    sa = DSA(xtr, ytr)
    for _ in range(3):          # eager launch, graph capture, graph replay
        got = sa(xte, pte)
        assert np.array_equal(got, want["dsa"])
        assert np.array_equal(sa.last_winner_index, want["idx_a"])
        assert np.array_equal(sa.last_dist_a, want["dist_a"]) and np.array_equal(sa.last_dist_b, want["dist_b"])


# pool items of 1, 2 and 3 train tiles; class sizes that are not multiples of 128 leave partial last tiles, and a
# CTA drawing successive pool items of one query tile keeps it resident
@pytest.mark.parametrize("pool_tiles", [1, 2, 3])
def test_dsa_pool_items_match_oracle(monkeypatch, pool_tiles):
    _dsa_case(monkeypatch, pool_tiles, n_train=9000, n_test=1500, classes=3, d=128, seed=31 + pool_tiles)


# purely static lists: consecutive static items of one CTA share the query tile
def test_dsa_static_items_match_oracle(monkeypatch):
    _dsa_case(monkeypatch, 4, n_train=7001, n_test=2000, classes=4, d=96, seed=41, pool_frac=0.0)


def test_dsa_mixed_class_tiles_match_oracle(monkeypatch):
    """A small batch over many classes: query tiles hold several classes, so the stage-2 launch masks each query's
    own class inside the tile (the EXCL instantiation)."""
    _dsa_case(monkeypatch, 2, n_train=6000, n_test=150, classes=12, d=64, seed=43)
