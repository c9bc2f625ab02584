"""Cost of dsm_frame_raw_cloud (publish_raw_pointcloud on the device) at 1226x370 and 1280x720.

Per size: the k_raw_cloud kernel time from torch.profiler's CUDA activity (a run of its own), the kernel's achieved
bandwidth on the 21 B/px model (5 B/px in: depth + gray; 16 B/px out) against the H100 SXM data sheet's 3.35 TB/s,
and the latency of the whole synchronising call (kernel + 16 B/px D2H into pageable memory) from a host clock,
profiler off.  The card name and power limit are read in the same run.
Usage: python tools/measure_raw_cloud.py [--iters N] [--out DIR]   (writes DIR/raw_cloud.json when --out is given)
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402

BYTES_PER_PX = 21
HBM_PEAK_GBS = 3350.0
POSE7 = np.array([0.4, -1.25, 2.5, 0.12, -0.31, 0.05, -0.93])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def measure(cam, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=200000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    pose = synth.pose_stream(3)
    g, d = synth.make_frame(cam, 3, pose)
    ctx.fuse_frame_resident(0, g, d, pose)
    npx = cam.width * cam.height
    out = np.zeros(npx, capi.POINT_DTYPE)
    n = capi.ctypes.c_int(0)
    p7 = np.ascontiguousarray(POSE7)

    def call():
        ctx._ck(ctx.lib.dsm_frame_raw_cloud(ctx.h, 0, p7.ctypes.data, out.ctypes.data, npx, capi.ctypes.byref(n)))

    for _ in range(20):   # warm-up: allocation of the output buffer, first launches, pages of `out`
        call()
    lat = []
    for _ in range(iters):
        t0 = time.perf_counter()
        call()
        lat.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "k_raw_cloud" in e.name]
    ker_us = float(np.median([e.device_time for e in kern])) if kern else float("nan")
    copy = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy DtoH" in e.name]
    copy_us = float(np.median([e.device_time for e in copy])) if copy else float("nan")
    ctx.close()
    gbs = npx * BYTES_PER_PX / (ker_us * 1e-6) / 1e9
    return dict(size=f"{cam.width}x{cam.height}", points=npx, kernel_us_median=ker_us, kernel_launches_seen=len(kern),
                kernel_gbs_21B_per_px=gbs, kernel_share_of_3350_gbs=gbs / HBM_PEAK_GBS,
                d2h_copy_us_median=copy_us,
                call_ms_median=1e3 * float(np.median(lat)), call_ms_min=1e3 * float(np.min(lat)), call_ms_max=1e3 * float(np.max(lat)),
                iters=iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_raw_cloud: no CUDA device (nothing is measured without one)")
    res = dict(card=card(), results=[measure(c, a.iters) for c in (synth.KITTI, synth.HD)])
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "raw_cloud.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
