"""Where does a resident single-frame stream spend its time?  Per-call host time and device time of dsm_fuse_frame_resident
(a one-frame dsm_fuse_stream_resident: phase 1 and phase 2 are two graphs per frame, on two streams) with and without
CUDA graphs.   python tools/stream_probe.py"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402

cam = synth.KITTI
T = 16
fr = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(T)]
tg = torch.from_numpy(np.stack([f[0] for f in fr])).pin_memory()
td = torch.from_numpy(np.stack([f[1] for f in fr])).pin_memory()
hg, hd = tg.numpy(), td.numpy()
P = np.stack([synth.pose_stream(t) for t in range(T)])
for graphs in ("1", "0"):
    os.environ["DSM_GRAPHS"] = graphs
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=2_000_000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for t in range(4):
        ctx.fuse_frame_resident(t // 4, hg[t], hd[t], P[t])
    ctx.sync()
    host = []
    t0 = time.perf_counter()
    for rep in range(3):
        for t in range(4, T):
            a = time.perf_counter()
            ctx.fuse_frame_resident((rep * T + t) // 4, hg[t], hd[t], P[t])
            host.append(time.perf_counter() - a)
    t1 = time.perf_counter()
    ctx.sync()
    t2 = time.perf_counter()
    n = 3 * (T - 4)
    print(f"graphs={graphs}: {n} frames, enqueue {1e3 * (t1 - t0) / n:.3f} ms/frame (median call {1e3 * np.median(host):.3f}, max {1e3 * max(host):.3f}), "
          f"drain {1e3 * (t2 - t1):.3f} ms, total {1e3 * (t2 - t0) / n:.3f} ms/frame, pool {ctx.pool_size()}", flush=True)
    ctx.close()
