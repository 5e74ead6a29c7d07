"""Per-tile phase times of the DSA filter kernel at C2, from the kernel's clock64 stamps (block 0).

    python tools/filter_timeline.py [--tiles 512] [--root DIR] [--json OUT]

Runs C2's stage-1 (same-class columns) and stage-2 (other-class columns) searches once each with
`tip_debug_timeline` on and turns the stamps of block 0 into per-tile phases, in SM clocks:
  mma      consumer: first MMA issue of the tile (slot 0) -> its MMAs retired (slot 1), including the
           waits for the tile's chunks to land
  epilogue consumer: MMAs retired (slot 1) -> reduction done and events handed to the drain (slot 7)
  drain    drain warps: the tile's events received (slot 11) -> staged / emitted (slot 12); a build without
           drain warps reports null
  period   consumer: tile start -> next tile start (slot 0 to slot 0)
  lead     producer ahead of the consumers: producer starts loading the tile (slot 8) -> consumer starts
           issuing it (slot 0); large means the ring is full and the consumers are the limit
  load     producer: first -> last TMA issue of the tile (slot 8 -> slot 10), including waits for free stages
  ev_wait  consumer: the epilogue's wait for a free event mailbox (slot 1 -> slot 2), i.e. for the drain to have
           taken the events of two tiles back; part of `epilogue`
p50 / p90 over the tiles of block 0.  `chunk_pass` is, per consumer warp, the share of block 0's tiles on which the
warp took the chunk pass (some row's tile minimum inside its window; slot 3 holds one bit per warp).  Stage 2 runs here from freshly packed queries, so its running minima start
at +inf; bench.py's stage 2 starts from the bounds stage 1 found, so fewer of its tiles reach the event path.
`search_ms` times the whole search call (query packing, the filter launch, the re-rank), not the filter alone.
`--root` runs the package found in another tree (e.g. a build of an earlier commit), so that two versions can be
compared with the same tool.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=512)
    ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch

    from oracle import np_oracle
    from simple_tip_b200 import _lib
    from simple_tip_b200 import engine as E
    from simple_tip_b200.core.surprise import DSA

    xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(60000, 10000, 128, 10, seed=2)
    sa = DSA(xtr, ytr)
    eng = sa._engine
    order, q_off = E.class_layout(pte, 10)
    x = E.to_device(xte, eng.dev).index_select(0, torch.from_numpy(order).to(eng.dev))
    qc = torch.from_numpy(pte[order].astype(np.int32)).to(eng.dev)
    lib = _lib.load()
    w = eng.gather(eng.search(x, qc, q_off, _lib.RANGE_SAME_CLASS)[1])
    out = {"gpu": torch.cuda.get_device_name(0)}
    for name, mode, q in (("stage1_same_class", _lib.RANGE_SAME_CLASS, x), ("stage2_other_classes", _lib.RANGE_OTHER_CLASSES, w)):
        for _ in range(2):
            eng.search(q, qc, q_off, mode)
        torch.cuda.synchronize()
        buf = torch.zeros((args.tiles, 16), dtype=torch.int64, device=eng.dev)
        lib.tip_debug_timeline(C.c_void_p(buf.data_ptr()), args.tiles)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        eng.search(q, qc, q_off, mode)
        ev1.record()
        torch.cuda.synchronize()
        lib.tip_debug_timeline(None, 0)
        t = buf.cpu().numpy()
        t = t[(t[:, 0] > 0) & (t[:, 1] > 0) & (t[:, 7] > 0) & (t[:, 8] > 0) & (t[:, 10] > 0)]
        ph = {"mma": t[:, 1] - t[:, 0], "epilogue": t[:, 7] - t[:, 1], "period": np.diff(t[:, 0]),
              "lead": t[:, 0] - t[:, 8], "load": t[:, 10] - t[:, 8]}
        ph["ev_wait"] = (t[:, 2] - t[:, 1])[t[:, 2] > 0]
        d = buf.cpu().numpy()
        d = d[(d[:, 11] > 0) & (d[:, 12] > 0)]
        ph["drain"] = d[:, 12] - d[:, 11]
        rec = {"tiles": int(len(t)), "search_ms": ev0.elapsed_time(ev1)}
        for k, v in ph.items():
            rec[k] = {"p50": float(np.percentile(v, 50)), "p90": float(np.percentile(v, 90))} if len(v) else None
        q_rows, t_rows = C.c_int32(), C.c_int32()
        lib.tip_nn_filter_tile(128, C.byref(q_rows), C.byref(t_rows))
        warps = q_rows.value // 16          # one consumer warp per 16 query rows of a tile
        rec["chunk_pass"] = [round(float(((t[:, 3] >> w) & 1).mean()), 3) for w in range(warps)] if len(t) else None
        out[name] = rec
        print(name, json.dumps(rec), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
