"""Cost of the resident pool's fuse_map post-step, seen from the caller: dsm_fuse_frame_resident and a 16-frame
dsm_fuse_stream_resident on pools of about 6 k, 100 k, 1 M and 2 M surfels, 1226x370 frames.

Before every timed call the pool is uploaded again (untimed): surfels spread in front of the camera, update_times 10 so
that no stability rule removes them, and 0.5 % of the slots dead, which is about what k_fuse kills per frame on the
benchmark's stream.  Each frame adds its new surfels (a few thousand).  Time: host clock around the call and a
dsm_pool_size that synchronises; median of --iters.  --lib times another build of the library (an A/B runs this
script once per build, alternately, in one job).  The card name and power limit are read in the same run.
Usage: python tools/measure_pool_poststep.py [--lib PATH] [--iters N] [--sizes a,b,...] [--out FILE]
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

CHUNK = 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_pool(n, rng):
    p = np.zeros(n, SURFEL_DTYPE)
    p["px"] = rng.uniform(-20, 20, n)
    p["py"] = rng.uniform(-3, 3, n)
    p["pz"] = rng.uniform(2, 60, n)
    p["nz"] = -1.0
    p["size"], p["weight"], p["color"] = 0.05, 1.0, 100.0
    p["update_times"] = 10
    p["last_update"] = 0
    p["update_times"][rng.random(n) < 0.005] = 0
    return p


def median_ms(call, before, iters):
    for _ in range(3):
        before()
        call()
    lat = []
    for _ in range(iters):
        before()
        t0 = time.perf_counter()
        call()
        lat.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(lat)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--sizes", default="6000,100000,1000000,2000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.lib:
        capi.LIB_PATH = os.path.abspath(a.lib)
    cam = synth.KITTI
    rng = np.random.default_rng(0)
    fr = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(CHUNK)]
    gray = np.stack([f[0] for f in fr])
    depth = np.stack([f[1] for f in fr])
    poses = np.stack([synth.pose_stream(t) for t in range(CHUNK)])
    res = {"card": card(), "lib": a.lib or "in-tree", "frame": f"{cam.width}x{cam.height}", "sizes": {}}
    for n in (int(s) for s in a.sizes.split(",")):
        pool = make_pool(n, rng)
        ctx = capi.Context(cam, max_batch=2 * CHUNK, max_local_surfels=n + (CHUNK + 2) * ctx_seeds(cam))
        up = lambda: ctx.pool_upload(pool)
        one = lambda: (ctx.fuse_frame_resident(0, gray[0], depth[0], poses[0]), ctx.pool_size())
        many = lambda: (ctx.fuse_stream_resident(list(range(CHUNK)), gray, depth, poses), ctx.pool_size())
        up()
        one()
        grown = ctx.pool_size()
        res["sizes"][str(n)] = {"dead_slots": int((pool["update_times"] == 0).sum()), "size_after_one_frame": grown,
                                "frame_ms": median_ms(one, up, a.iters),
                                "stream16_ms": median_ms(many, up, a.iters)}
        ctx.close()
        print(n, res["sizes"][str(n)], flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


def ctx_seeds(cam):
    from densesurfelmapping_b200.elements import num_seeds
    return num_seeds(cam.width, cam.height)


if __name__ == "__main__":
    main()
