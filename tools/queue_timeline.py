"""Developer aid (needs a GPU): where a scan's time goes in the QUEUED path (kb_pipeline_register_frames), from the light
in-kernel stamps (phase boundaries only), once with the front-end prefetch on and once with it off, on the same scans
(two pipelines primed alike). Prefetch off isolates what the next scan's front end costs the ICP team beside it.
The gap between two launches is split at the launch boundary: last CTA of launch k left -> first CTA of launch k + 1
entered (negative: launch k + 1 was placed while launch k was still ending), and first CTA entered -> every CTA past the
prologue (state read, veto decided).
usage: python tools/queue_timeline.py [prime=100] [frames=40]"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kiss_icp_b200 as K
from kiss_icp_b200 import _native as N, synthetic

prime = int(sys.argv[1]) if len(sys.argv) > 1 else 100
frames = int(sys.argv[2]) if len(sys.argv) > 2 else 40
L = synthetic.kitti_shape(seed=0, device="cuda")
scans = [L.scan_torch(k) for k in range(prime + frames)]


def stamps(fn, h, cols):
    n = N.sz(0)
    N.check(fn(h, None, 0, C.byref(n)))
    st = np.zeros((n.value, cols))
    N.check(fn(h, N.ptr(st), n.value, C.byref(n)))
    return st


def run(prefetch):
    g = K.KissICP(K.load_config())
    N.check(N.lib().kb_pipeline_debug_prefetch(g._h, int(prefetch)))
    raw = lambda ss: g._register_frames_raw([s[0].data_ptr() for s in ss], [s[0].shape[0] for s in ss], [None] * len(ss), [0] * len(ss), 2)
    raw(scans[:prime])
    N.check(N.lib().kb_pipeline_set_profiling(g._h, 2))  # phase boundaries only (KissICP.set_profiling turns on level 1)
    g.start_history(frames)
    raw(scans[prime:])
    st = stamps(N.lib().kb_pipeline_history_stamps, g._h, 20)
    gr = stamps(N.lib().kb_pipeline_history_grid_stamps, g._h, 3)
    return g, st, gr


us = lambda a: np.round(np.median(a) * 1e-3, 1)
for prefetch in (True, False):
    g, st, gr = run(prefetch)
    h = g.history()
    t = st[2:-1]  # steady part
    print(f"prefetch {'on' if prefetch else 'off'}: frames", len(t), "team", h[-1].team, "iterations (median)",
          np.median([x.iterations for x in h]), "last pose", g.last_pose[:3, 3].tolist())
    print("  kernel total", us(t[:, 6] - t[:, 0]), "| front end in the launch", us(t[:, 3] - t[:, 0]),
          "| start->lists done", us(t[:, 7] - t[:, 0]), "| lists done", us(t[:, 7] - t[:, 3]),
          "| lists->iterations done", us(t[:, 10] - t[:, 7]), "| prefetch done after lists", us(t[:, 11] - t[:, 7]) if prefetch else "-",
          "| iterations->result everywhere", us(t[:, 4] - t[:, 10]), "| map update", us(t[:, 5] - t[:, 4]), "| tail", us(t[:, 6] - t[:, 5]))
    print("  gap between kernels (CTA 0)", us(st[3:, 0] - st[2:-1, 6]), "| period", us(np.diff(st[2:, 0])))
    print("  launch boundary: last CTA of k left -> first CTA of k+1 entered", us(gr[3:, 0] - gr[2:-1, 2]),
          "| first CTA entered -> every CTA past the prologue", us(gr[3:, 1] - gr[3:, 0]),
          "| CTA 0 end stamp -> last CTA left", us(gr[2:-1, 2] - st[2:-1, 6]),
          "| last CTA of k left -> every CTA of k+1 past the prologue", us(gr[3:, 1] - gr[2:-1, 2]))
