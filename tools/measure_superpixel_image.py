"""Cost of dsm_frame_superpixel_image (FusionFunctions::debug_show on the device) at 1226x370 and 1280x720.

Per size: the k_superpixel_image kernel time and the D2H copy time from torch.profiler's CUDA activity (a run of its
own), the kernel's achieved bandwidth on a 4 B/px model (1 B/px of label codes in, 3 B/px of image out; the row below
and the plane records are cache hits and not counted) against the H100 SXM data sheet's 3.35 TB/s, and the latency of
the whole synchronising call (kernel + 3 B/px D2H) from a host clock, profiler off, into pageable and into pinned host
memory.  The card name and power limit are read in the same run.
Usage: python tools/measure_superpixel_image.py [--iters N] [--out DIR]   (writes DIR/superpixel_image.json with --out)
"""
import argparse
import ctypes
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

BYTES_PER_PX = 4
HBM_PEAK_GBS = 3350.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def latency(call, iters):
    for _ in range(20):   # warm-up: staging allocation, first launches, pages of the output
        call()
    lat = []
    for _ in range(iters):
        t0 = time.perf_counter()
        call()
        lat.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(lat)), 1e3 * float(np.min(lat)), 1e3 * float(np.max(lat))


def measure(cam, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=200000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    pose = synth.pose_stream(3)
    g, d = synth.make_frame(cam, 3, pose)
    ctx.fuse_frame_resident(0, g, d, pose)
    npx = cam.width * cam.height
    pitch = 3 * cam.width
    pageable = np.zeros((cam.height, pitch), np.uint8)
    pinned = torch.empty(cam.height * pitch, dtype=torch.uint8, pin_memory=True)

    def call_into(ptr):
        return lambda: ctx._ck(ctx.lib.dsm_frame_superpixel_image(ctx.h, 0, ctypes.c_void_p(ptr), pitch))

    call_pageable, call_pinned = call_into(pageable.ctypes.data), call_into(pinned.data_ptr())
    lat_pageable = latency(call_pageable, iters)
    lat_pinned = latency(call_pinned, iters)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call_pageable()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kern = [e.device_time for e in ev if "k_superpixel_image" in e.name]
    copy = [e.device_time for e in ev if "Memcpy" in e.name and "DtoH" in e.name]
    ker_us = float(np.median(kern)) if kern else float("nan")
    copy_us = float(np.median(copy)) if copy else float("nan")
    ctx.close()
    gbs = npx * BYTES_PER_PX / (ker_us * 1e-6) / 1e9
    return dict(size=f"{cam.width}x{cam.height}", pixels=npx, kernel_us_median=ker_us, kernel_launches_seen=len(kern),
                kernel_gbs_4B_per_px=gbs, kernel_share_of_3350_gbs=gbs / HBM_PEAK_GBS,
                d2h_copy_us_median=copy_us, d2h_copies_seen=len(copy),
                call_pageable_ms_median=lat_pageable[0], call_pageable_ms_min=lat_pageable[1], call_pageable_ms_max=lat_pageable[2],
                call_pinned_ms_median=lat_pinned[0], call_pinned_ms_min=lat_pinned[1], call_pinned_ms_max=lat_pinned[2],
                iters=iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_superpixel_image: no CUDA device (nothing is measured without one)")
    res = dict(card=card(), results=[measure(c, a.iters) for c in (synth.KITTI, synth.HD)])
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "superpixel_image.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
