"""Measure the terrain viewpoint job (dsm_viewpoint_enqueue_terrain, DESIGN.md §8.23) against the two paths a ground
planner takes without it.

Cases, each a terrain job (headroom 5, max step 1) on a loaded known field, its frontier job, and a terrain reach job
(host copy) from a random traversable cell (seeded):
  road        the synthetic road request of DESIGN.md §8.20 (tools/measure_reach_terrain.road), up = -2, 0.2 m;
  obstacles   320 x 320 and 1024 x 1024 z-up planes at 0.1 m: an occupied floor with 8 % of the columns unobserved and
              long walls with one gap each (tools/measure_reach_terrain.obstacles); the unobserved columns' borders are
              the frontier clusters.
Per case, the job names the first --clusters clusters, with 32 rotations (16 headings, level and pitched 0.3 rad
down), eye 4, a ring of radius 2..8 cells at stride 2, 256 samples, top_k 4, with reach, and a 6 m range with unknown
space blocking:
1. The job: host clock from dsm_viewpoint_enqueue_terrain to the end of dsm_viewpoint_wait on an idle stream, median
   and range of --reps, and the per-kernel device times of torch.profiler (CUDA activities, --launches jobs).  The
   result is checked equal to the host model.
2. The same reached candidates and rotations scored as gain views (dsm_gain_enqueue naming each cluster, in jobs of as
   many views as gain's work bound n_views (2 ceil(R / v) + 3)^3 <= 2^31 and --views allow): one pass timed, host clock
   around the enqueues and waits.
3. The host model (oracle/pyoracle_viewpoint_terrain) on the host copies of the state grid and the planes: one pass.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_viewpoint_terrain.py [--clusters 32] [--reps 10] [--out DIR]"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import card, spread  # noqa: E402
from measure_reach_terrain import HEADROOM, MAX_STEP, floored, obstacles, road  # noqa: E402
from ground_views import rotations  # noqa: E402
import pyoracle_gain as G  # noqa: E402
import pyoracle_reach as R  # noqa: E402
import pyoracle_reach_terrain as RT  # noqa: E402
import pyoracle_viewpoint as V  # noqa: E402
import pyoracle_viewpoint_terrain as VT  # noqa: E402

KERNELS = ("k_vp_score", "k_vp_candidates", "k_vp_select", "k_vp_clusters")
EYE = 4
RANGE = 6.0


def cases(rng):
    state, origin = road()
    yield "road", (state, origin, 0.2, -2)
    for n in (320, 1024):
        yield f"obstacles {n}", (floored(obstacles(n, rng)), np.zeros(3, np.int32), 0.1, 3)


def gain_views(terrain, voxel, fr, cl, rot, prm, cost):
    """The poses [R_r | t] and cluster of every reached candidate and rotation of the job, as gain views."""
    tinfo, level, status, _, clearance = terrain
    up = int(tinfo["up"])
    h0, h1 = RT.plane_axes(up)
    P, Q = int(tinfo["m"][h0]), int(tinfo["m"][h1])
    trav = R.traversable(status.reshape(1, Q, P), clearance.reshape(1, Q, P), prm.radius)[0]
    table = fr[0]
    off = V.offsets(prm)[:, :2]
    poses, names = [], []
    for c in cl:
        g = VT.centre_cell(table[c]["centroid"], [int(x) for x in tinfo["origin"]], voxel, up)[:2]
        for x, y in g + off:
            if 0 <= x < P and 0 <= y < Q and trav[y, x] and cost.reshape(Q, P)[y, x] != R.INF:
                t = VT.camera_point(int(y * P + x), terrain, voxel, EYE)
                for Rm in rot:
                    poses.append(np.concatenate([Rm.reshape(3, 3), t[:, None]], axis=1).reshape(12))
                    names.append(c)
    return np.array(poses).reshape(-1, 12), np.array(names, np.int32)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--clusters", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--views", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    res = {"card": name, "power_limit": power, "cases": []}
    rng = np.random.default_rng(1)
    for label, (state, origin, voxel, up) in cases(rng):
        nz, ny, nx = state.shape
        ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=1 << 12)
        ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
        ctx.field_enable(voxel, nx, ny, nz)
        ctx.views_enable(1, 1.0)
        ctx.terrain_enable(up)
        ctx.frontier_enable(4096, 1 << 22)
        ctx.reach_enable(1, 1, 4096)
        ctx.gain_enable(a.views)
        ctx.viewpoint_enable(a.clusters, 1 << 20)
        ctx.debug_field_load_state(state, origin)
        ctx.field_wait()
        ctx.terrain_enqueue(HEADROOM, MAX_STEP)
        terrain = ctx.terrain_wait()
        ctx.frontier_enqueue(1)
        fc, fv, _ = ctx.frontier_wait()
        h0, h1 = RT.plane_axes(up)
        P = int(terrain[0]["m"][h0])
        cells = np.flatnonzero(terrain[2].reshape(-1) == 2)
        c0 = int(rng.choice(cells))
        v = float(np.float32(voxel))
        start = [0.0, 0.0, 0.0]
        start[h0], start[h1] = (c0 % P + int(origin[h0]) + 0.5) * v, (c0 // P + int(origin[h1]) + 0.5) * v
        ctx.reach_enqueue_terrain(tuple(start), 0.0, 2, None, False, True)
        cost = ctx.reach_wait()[3]
        rot = rotations(up, 16, (0.0, -0.3))
        cam = G.Camera(synth.KITTI.fx, synth.KITTI.fy, synth.KITTI.cx, synth.KITTI.cy, synth.KITTI.width, synth.KITTI.height, RANGE, 1)
        cl = np.arange(min(len(fc), a.clusters), dtype=np.int32)
        prm = V.Params(2, 8, 0, 2, 256, 1, 4, 1, 0.0)
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, EYE)
        got = ctx.viewpoint_wait()
        t0 = time.perf_counter()
        want = VT.viewpoints(state, voxel, terrain, cam, rot, cl, prm, EYE, (fc, fv), cost)
        model_ms = (time.perf_counter() - t0) * 1e3
        equal = all(g.tobytes() == np.asarray(w).tobytes() for g, w in zip(got, want))
        lib, h = ctx.lib, ctx.h
        gc = capi._camera(cam)
        R9 = np.ascontiguousarray(rot)
        p = capi.DsmViewpointParams(*prm[:8], prm.radius, 0)

        def job():
            assert lib.dsm_viewpoint_enqueue_terrain(h, ctypes.byref(gc), R9.ctypes.data, len(R9), cl.ctypes.data, len(cl), ctypes.byref(p),
                                                     EYE) == 0
            assert lib.dsm_viewpoint_wait(h, None, None, None) == 0
        for _ in range(2):
            job()
        ts = []
        for _ in range(a.reps):
            ctx.sync()
            t0 = time.perf_counter()
            job()
            ts.append((time.perf_counter() - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.launches):
                job()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            key = next((n for n in KERNELS if n in e.key), "memcpy" if "Memcpy" in e.key else None)
            if key:
                kern[key] = kern.get(key, 0.0) + e.device_time_total / a.launches
        # the same candidates and rotations as gain views
        poses, names = gain_views(terrain, voxel, (fc, fv), cl, rot, prm, cost)
        ctx.gain_enqueue(cam, poses[:8], names[:8])
        ctx.gain_wait()
        m = 2 * int(np.ceil(np.float32(RANGE) / np.float32(voxel))) + 3
        chunk = min(a.views, G.MAX_WORK // m ** 3)
        ctx.sync()
        t0 = time.perf_counter()
        for i in range(0, len(poses), chunk):
            ctx.gain_enqueue(cam, poses[i:i + chunk], names[i:i + chunk])
            ctx.gain_wait()
        gain_ms = (time.perf_counter() - t0) * 1e3
        recs = got[1]
        r = {"case": label, "grid": [nx, ny, nz], "up": up, "clusters": len(cl), "clusters_table": len(fc),
             "n_reached": int(recs["n_reached"].sum()), "n_viewpoints": int(recs["n_viewpoints"].sum()), "equal_to_model": equal,
             "job_ms": spread(ts), "kernels_us_per_job": kern, "gain_views": len(poses), "gain_jobs": -(-len(poses) // chunk), "gain_views_ms": gain_ms,
             "host_model_ms": model_ms}
        res["cases"].append(r)
        print(json.dumps(r), flush=True)
        ctx.close()
    print(json.dumps({"card": name, "power_limit": power}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_viewpoint_terrain.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
