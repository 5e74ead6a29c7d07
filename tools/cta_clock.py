"""Per-CTA start/end times (globaltimer) of the resident-query filter kernel at C2 (bring-up tool)."""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import np_oracle  # noqa: E402
from simple_tip_b200 import _lib  # noqa: E402
from simple_tip_b200 import engine as E  # noqa: E402
from simple_tip_b200.core.surprise import DSA  # noqa: E402

xtr, ytr, xte, pte, _ = np_oracle.synth_clusters(60000, 10000, 128, 10, seed=2)
sa = DSA(xtr, ytr)
eng = sa._engine
order, q_off = E.class_layout(pte, 10)
x = E.to_device(xte, eng.dev).index_select(0, torch.from_numpy(order).to(eng.dev))
qc = torch.from_numpy(pte[order].astype(np.int32)).to(eng.dev)
lib = _lib.load()
_, pos, _, _ = eng.search(x, qc, q_off, _lib.RANGE_SAME_CLASS)
w = eng.gather(pos)


def distinct():
    # DSA's stage 2 as dsa_distances runs it: once per distinct winner, live-bounded work list drawn from the pool
    rows, state, slot_class, live_end, _, _ = eng.distinct_winners(pos, q_off)
    eng.search(rows, slot_class, q_off, _lib.RANGE_OTHER_CLASSES, prepacked=state, live_end=live_end)


runs = [("other classes, every input", _lib.RANGE_OTHER_CLASSES, lambda: eng.search(w, qc, q_off, _lib.RANGE_OTHER_CLASSES)),
        ("other classes, distinct winners", _lib.RANGE_OTHER_CLASSES, distinct),
        ("same class", _lib.RANGE_SAME_CLASS, lambda: eng.search(x, qc, q_off, _lib.RANGE_SAME_CLASS))]
for label, mode, run in runs:
    for _ in range(2):
        run()
    buf = torch.zeros((320, 4), dtype=torch.int64, device=eng.dev)     # rows 0..255: per-CTA records, 256..: entry times
    lib.tip_debug_cta_clock(C.c_void_p(buf.data_ptr()))
    E.PROFILE = []
    run()
    torch.cuda.synchronize()
    prof, E.PROFILE = E.PROFILE, None
    lib.tip_debug_cta_clock(None)
    raw = buf.cpu().numpy()
    entry = raw.reshape(-1)[1024:1024 + 148]
    t = raw[:256]
    pro = (t[:148, 0] - entry) / 1e3
    print(f"{label}: kernel entry -> post-allocation timestamp per CTA: min {pro.min():.2f} p50 {np.median(pro):.2f} max {pro.max():.2f} us; "
          f"entry skew across CTAs {(entry.max() - entry.min()) / 1e3:.2f} us; first entry -> last CTA end {(t[:148, 1].max() - entry.min()) / 1e3:.1f} us; "
          f"event-timed launches: {[(k, round(a.elapsed_time(b) * 1e3, 1)) for k, _, a, b in prof] if prof else None}")
    t = t[t[:, 1] > 0]
    items = t[:, 3] & 0xffffffff
    smid = t[:, 3] >> 32
    t0 = t[:, 0].min()
    start, end = (t[:, 0] - t0) / 1e3, (t[:, 1] - t0) / 1e3
    dur = end - start
    print(f"{label}: {len(t)} CTAs; kernel span {end.max():.1f} us; CTA start skew max {start.max():.1f} us; "
          f"CTA duration min {dur.min():.1f} p50 {np.median(dur):.1f} p90 {np.percentile(dur, 90):.1f} max {dur.max():.1f} us")
    print(f"  tiles per CTA min {t[:, 2].min()} p50 {np.median(t[:, 2]):.0f} max {t[:, 2].max()}; items per CTA min {items.min()} max {items.max()}")
    print(f"  ns per tile: min {np.min(dur * 1e3 / t[:, 2]):.0f} p50 {np.median(dur * 1e3 / t[:, 2]):.0f} max {np.max(dur * 1e3 / t[:, 2]):.0f}")
    slow = np.argsort(-dur)[:8]
    print("  slowest CTAs (cta, smid, us, tiles, items):", [(int(i), int(smid[i]), round(float(dur[i]), 1), int(t[i, 2]), int(items[i])) for i in slow])
    fast = np.argsort(dur)[:8]
    print("  fastest CTAs (cta, smid, us, tiles, items):", [(int(i), int(smid[i]), round(float(dur[i]), 1), int(t[i, 2]), int(items[i])) for i in fast])
