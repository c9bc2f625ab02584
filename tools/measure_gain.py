"""Measure the gain jobs (dsm_gain_*, DESIGN.md §8.12) against the host path a planner uses without them.

1. Known fields of tools/measure_field_known.py's scene (eight 1226x370 frames captured into 256 slots) at 0.2 m, for
   every --grids grid: the state grid is taken once and loaded (dsm_debug_field_load_state) into one context, a frontier
   job and a reach job from the scene's centre give the viewpoints, and the views are eight yaws at each reached
   viewpoint (cycled, with a 15-degree downward tilt on every other round of eight, to --views each).  For every
   --views count and --ranges range (in voxels), with the 1226x370 camera and clusters named: the latency, host clock
   from dsm_gain_enqueue to the end of dsm_gain_wait on an idle stream (median, min-max of --reps); a count whose work
   bound n_views (2 ceil(R / v) + 3)^3 passes 2^31 voxels runs as the fewest equal requests that pass it, and the
   latency covers all of them.  Kernel times from torch.profiler in a run of their own.  Against that, the host path:
   the state grid's D2H copy (a host-copy known request minus a resident one, both waited for) and the numpy model
   (oracle/pyoracle_gain) on --host-views of the views, per view.
2. The node drive of tools/measure_node.py (tools/measure_gain.cpp), modes alternating on fresh nodes, --rounds rounds,
   a 320x320x40 known field read after every fuse: r with frontiers(1) and reach(with_frontiers) after every fuse; g
   with view_gain() as well, eight yaws at each of the first 64 reached viewpoints, clusters named, at 25 voxels.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_gain.py [--frames 320] [--rounds 3] [--out DIR]"""
import argparse
import json
import math
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import build_harness, card, images, kernel_us, messages, run_harness, spread, write_drive  # noqa: E402
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
import pyoracle_gain  # noqa: E402

KERNELS = ["k_gain_slots", "k_gain_init", "k_gain_views"]
CAM = synth.KITTI


def timed(fn, reps, ctx):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def yaw_views(points, n):
    """n poses: eight yaws about the world z axis at each point, cycled; every other round of eight tilts 15 degrees."""
    out = []
    for i in range(n):
        p = points[(i // 8) % len(points)]
        a, tilt = 0.25 * math.pi * (i % 8), np.deg2rad(15.0) * ((i // (8 * len(points))) % 2)
        f = np.array([math.cos(a) * math.cos(tilt), math.sin(a) * math.cos(tilt), -math.sin(tilt)])
        r = np.array([math.sin(a), -math.cos(a), 0.0])
        d = np.cross(f, r)
        out.append(np.concatenate([np.stack([r, d, f], 1), np.asarray(p, np.float64)[:, None]], 1).reshape(12))
    return np.array(out)


def requests(n, R):
    m = 2 * math.ceil(float(np.float32(R)) / float(np.float32(VOXEL))) + 3
    k = max(1, math.ceil(n * m ** 3 / pyoracle_gain.MAX_WORK))
    return [(i * n // k, (i + 1) * n // k) for i in range(k)]


def measure(state, origin, centre, grid, a, cp):
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(4096, 1 << 20)
    ctx.reach_enable(4096, 1 << 18, 4096)
    ctx.gain_enable(max(a.views))
    ctx.debug_field_load_state(state, origin)
    ctx.field_wait()
    ctx.frontier_enqueue(1)
    fc, fv, _ = ctx.frontier_wait()
    ctx.reach_enqueue(centre, VOXEL, 2, None, True)
    _, targets, _, _ = ctx.reach_wait()
    ok = targets["status"] == 0
    vp = targets["viewpoint"][ok]
    nz, ny, nx = state.shape
    pts = pyoracle_gain.centres(np.stack([vp % nx, vp // nx % ny, vp // (nx * ny)], 1), origin, VOXEL) if len(vp) else [centre]
    clusters_of = (np.flatnonzero(ok) if len(vp) else np.array([-1])).astype(np.int32)
    r = {"grid": grid, "clusters": len(fc), "reached_viewpoints": int(len(vp)), "state_copy_ms": cp, "jobs": []}
    for R_vox in a.ranges:
        R = R_vox * VOXEL
        gc = pyoracle_gain.Camera(CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.width, CAM.height, R, 1)
        for n in a.views:
            poses = yaw_views(pts, n)
            cl = np.array([clusters_of[(i // 8) % len(clusters_of)] for i in range(n)], np.int32)
            parts = requests(n, R)

            def job():
                out = []
                for lo, hi in parts:
                    ctx.gain_enqueue(gc, poses[lo:hi], cl[lo:hi])
                    out.append(ctx.gain_wait()[1])
                return np.concatenate(out)
            g = job()
            e = {"max_range_voxels": R_vox, "views": n, "requests": len(parts), "latency_ms": timed(job, a.reps, ctx),
                 "frustum_voxels_per_view": float(g["n_frustum"].mean()), "seen_per_view": float((g["n_free"] + g["n_unknown"] + g["n_occupied"]).mean()),
                 "frontier_seen_per_view": float(g["n_frontier"].mean())}
            per = kernel_us(lambda: [job() for _ in range(a.launches)], KERNELS)
            e["kernels_us"] = {k: sum(v) / a.launches for k, v in per.items() if v}
            if n == a.views[0]:
                h = min(a.host_views, n)
                t0 = time.perf_counter()
                _, want = pyoracle_gain.gains(state, origin, VOXEL, gc, poses[:h], cl[:h], (fc, fv))
                e["host_model_ms_per_view"] = (time.perf_counter() - t0) * 1e3 / h
                assert want.tobytes() == g[:h].tobytes(), "device and model differ"
            r["jobs"].append(e)
            print(json.dumps(e), flush=True)
    ctx.close()
    return r


def node_drive(n_frames, rounds, grid):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_harness(tmp, "measure_gain")
        ff, fs = write_drive(tmp, images(), messages(n_frames))
        times = {m: [] for m in "rg"}
        last = {}
        for _ in range(rounds):
            for m in "rg":
                last[m] = run_harness(exe, ff, fs, [m, VOXEL, *grid, MAX_VIEWS, MAX_RANGE, 25 * VOXEL])
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "views_per_frame": last["g"]["views"] / n_frames,
            "ms_per_frame": {m: spread(times[m]) for m in "rg"}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["320x320x40", "512x512x64"])
    ap.add_argument("--views", type=int, nargs="+", default=[16, 256, 4096])
    ap.add_argument("--ranges", type=int, nargs="+", default=[25, 50])
    ap.add_argument("--host-views", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--node-grid", default="320x320x40")
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "camera": [CAM.width, CAM.height], "known": []}
    for gs in a.grids:
        grid = tuple(int(x) for x in gs.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)

        def field(host):
            ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses, host_copy=host)
            ctx.field_wait()
        ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses)
        origin = ctx.field_wait()[1]
        state = ctx.field_state()[0].copy()
        cp = {"host_copy": timed(lambda: field(True), a.reps, ctx), "resident": timed(lambda: field(False), a.reps, ctx)}
        ctx.close()
        res["known"].append(measure(state, origin, c, grid, a, cp))
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, tuple(int(x) for x in a.node_grid.split("x")))
        print(json.dumps(res["node_drive"]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_gain.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
