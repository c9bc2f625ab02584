"""Measure the known-space field (dsm_views_*, dsm_field_enqueue_known, DESIGN.md §8.9) against the plain field.

A 1226x370 context fuses eight synthetic frames once; each is captured into 32 of 256 slots, and view j sits at the
pose of frame j % 8 moved across and along the road, so that the views overlap the way a drive's keyframes do.  For
every --grids grid at 0.2 m and every --views count (the first N slots), centred on frame 4's camera:
1. Latency: host clock from the enqueue to the end of dsm_field_wait (host copy, through the C calls), median of --reps
   on an idle stream, for dsm_field_enqueue and dsm_field_enqueue_known.
2. k_field_carve from torch.profiler (CUDA activities, --launches requests), with rays and voxel visits per second.  The
   visits are counted on the host by oracle/pyoracle_field_known's walk of the same rays (whole segments; the kernel
   skips only rays that cannot reach the grid).
3. The node drive of tools/measure_node.py (1226x370, --frames frames) through dsm::SurfelMapNode
   (tools/measure_field_known.cpp), modes alternating on fresh nodes, --rounds rounds, a 320x320x40 field at 0.2 m read
   right after every fuse: p the plain field; k known space as well (256 slots, rays cut at 40 m), its state read too.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_field_known.py [--frames 320] [--rounds 3] [--out DIR]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_publish import CAM, card, spread, write_drive  # noqa: E402
import pyoracle_field_known  # noqa: E402

VOXEL, MAX_RANGE, MAX_VIEWS = 0.2, 40.0, 256


def pose12(p16):
    return np.asarray(p16, np.float64).reshape(4, 4).T[:3, :4].reshape(12).copy()


def scene():
    """The context with 256 captured slots, the views' poses, their rays (for counting) and the centre."""
    cam = synth.KITTI
    ctx = capi.Context(cam, max_batch=16, max_local_surfels=1 << 18)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    imgs = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(8)]
    ctx.fuse_stream_resident(list(range(8)), np.stack([g for g, _ in imgs]), np.stack([d for _, d in imgs]),
                             np.stack([synth.pose_stream(t) for t in range(8)]))
    rays = [pyoracle_field_known.capture(ctx.seeds(f)) for f in range(8)]   # one run of 8 frames: frame slots 0..7
    poses, views = [], []
    for j in range(MAX_VIEWS):
        P = pose12(synth.pose_stream(j % 8))
        P[3] += 0.35 * (j // 8 % 8) - 1.2
        P[11] += 0.8 * (j // 64)
        poses.append(P)
        views.append((rays[j % 8], P))
    return ctx, np.array(poses), views, pose12(synth.pose_stream(4))[[3, 7, 11]]


def visits(views):
    count = [0]

    def visit(r, ijk, end):
        count[0] += len(r)
    a, b = [], []
    for rays, P in views:
        s = pyoracle_field_known.segments(rays, P, MAX_RANGE)
        a.append(s[0])
        b.append(s[1])
    pyoracle_field_known.walk(np.concatenate(a), np.concatenate(b), VOXEL, visit)
    return count[0]


def build_driver(tmp):
    exe = os.path.join(tmp, "measure_field_known")
    pkg = os.path.join(ROOT, "densesurfelmapping_b200")
    subprocess.run(["g++", "-std=c++11", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tools", "measure_field_known.cpp"),
                    "-o", exe, "-L", pkg, "-ldsm_b200", f"-Wl,-rpath,{pkg}"], check=True)
    return exe


def run_mode(exe, ff, fs, mode, grid):
    args = [exe, str(CAM.width), str(CAM.height)] + [repr(float(v)) for v in (CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.far, CAM.near)]
    args += ["10", ff, fs, mode, repr(VOXEL)] + [str(n) for n in grid] + [str(MAX_VIEWS), repr(MAX_RANGE)]
    r = subprocess.run(args, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"measure_field_known mode {mode} exited {r.returncode}: {r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def node_drive(n_frames, rounds, grid):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_driver(tmp)
        ff, fs = write_drive(tmp, n_frames)
        times = {m: [] for m in "pk"}
        last = {}
        for _ in range(rounds):
            for m in "pk":
                last[m] = run_mode(exe, ff, fs, m, grid)
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "voxel": VOXEL, "views_at_end": last["k"]["views"],
            "free_per_field": last["k"]["free"] / max(last["k"]["fields"], 1), "ms_per_frame": {m: spread(times[m]) for m in "pk"}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--views", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--node-grid", default="320x320x40")
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "max_range": MAX_RANGE, "fields": []}
    counts = {}
    for g in a.grids:
        grid = tuple(int(x) for x in g.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)
        for n in a.views:
            slots = list(range(n))
            if n not in counts:
                counts[n] = {"rays": int(sum(len(v[0]) for v in views[:n])), "visits": visits(views[:n])}

            # the C calls, so that the host's numpy copy of the grid stays out of the latency
            lib, h, cc = ctx.lib, ctx.h, (ctypes.c_double * 3)(*c)
            sl, ps = np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(poses[:n])

            def plain():
                assert lib.dsm_field_enqueue(h, cc, 5) == 0 and lib.dsm_field_wait(h, None, None, None) == 0

            def known():
                assert lib.dsm_field_enqueue_known(h, cc, 5, sl.ctypes.data, ps.ctypes.data, n, 1) == 0
                assert lib.dsm_field_wait(h, None, None, None) == 0
            lat = {}
            for key, fn in (("plain", plain), ("known", known)):
                for _ in range(3):
                    fn()
                ts = []
                for _ in range(a.reps):
                    ctx.sync()
                    t0 = time.perf_counter()
                    fn()
                    ts.append((time.perf_counter() - t0) * 1e3)
                lat[key] = spread(ts)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.launches):
                    known()
                torch.cuda.synchronize()
            rows = [k for k in prof.key_averages() if "k_field_carve" in k.key]
            launches = sum(k.count for k in rows)
            if launches != a.launches:
                raise RuntimeError(f"profiler saw {launches} launches of k_field_carve, expected {a.launches}")
            us = sum(k.device_time_total for k in rows) / launches
            r = {"grid": grid, "views": n, "latency_ms": lat, "carve_us": us, **counts[n],
                 "rays_per_s": counts[n]["rays"] / (us * 1e-6), "visits_per_s": counts[n]["visits"] / (us * 1e-6)}
            res["fields"].append(r)
            print(json.dumps(r), flush=True)
        ctx.close()
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, tuple(int(x) for x in a.node_grid.split("x")))
        print(json.dumps(res["node_drive"]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_field_known.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
