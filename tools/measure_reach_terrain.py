"""Measure the terrain reach job (dsm_reach_enqueue_terrain, DESIGN.md §8.21) against the path a ground planner takes
without it.

Cases, each a terrain job (headroom 5, max step 1) on a loaded known field, then terrain reach jobs from one start to
three goals on its plane (the start the traversable cell nearest one corner; the goals the reached cells farthest from
it, nearest the middle and nearest the next corner, by Dijkstra on the host):
  road        the synthetic road request of DESIGN.md §8.20 (eight fused synthetic KITTI frames in 256 captured views
              moved across and along the road, 0.2 m, 64 x 20 x 128 voxels ahead of the first camera), up = -2;
  obstacles   320 x 320 and 1024 x 1024 z-up planes: an occupied floor with 8 % of the columns unobserved (no support)
              and long walls with one gap each;
  serpentine  a 256 x 256 z-up plane of walls every fourth row, open at alternating ends.
Per case and per round cap in --caps (max_rounds of dsm_reach_enable):
1. Latency: host clock from dsm_reach_enqueue_terrain to the end of dsm_reach_wait (through the C calls), median and
   range of --reps on an idle stream, with the rounds run and whether the job converged.
2. Per-kernel device times from torch.profiler (CUDA activities, --launches jobs): k_reach_round, k_reach_settle, the
   init, target and path kernels and the result's D2H copy.
3. The host alternative: the terrain planes a planner needs (status and clearance, 5 B per cell) copied device to host
   (pinned, torch), then scipy's Dijkstra on the 8-connected 10/14 graph (oracle/pyoracle_reach.dijkstra).
--lib runs the same cases on another build of the library (to compare tile shapes); the card's name and power limit
are read in the same run.  Fails without a GPU.
Usage: python tools/measure_reach_terrain.py [--caps 16 64 256] [--reps 30] [--lib PATH] [--out DIR]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import card, spread  # noqa: E402
import pyoracle_reach as R  # noqa: E402
import pyoracle_reach_terrain as RT  # noqa: E402

KERNELS = ("k_reach_round", "k_reach_settle", "k_reach_init", "k_reach_start", "k_reach_reached", "k_reach_targets",
           "k_reach_records", "k_reach_paths")
HEADROOM, MAX_STEP = 5, 1


def floored(walls, n_up=8):
    """A z-up state grid [n_up][Q][P]: an occupied floor under free space, every voxel unknown where `walls` holds."""
    Q, P = walls.shape
    st = np.full((n_up, Q, P), R.FREE, np.uint8)
    st[0] = R.OCCUPIED
    st[:, walls] = R.UNKNOWN
    return st


def obstacles(n, rng):
    w = rng.random((n, n)) < 0.08
    for j, x in enumerate(range(n // 4, n, n // 4)):
        w[:, x] = True
        gap = (j * 7919) % (n - 8)
        w[gap:gap + 6, x] = False
    return w


def serpentine(n):
    w = np.zeros((n, n), bool)
    for i, q in enumerate(range(3, n - 1, 4)):
        w[q, :] = True
        w[q, n - 1 if i % 2 == 0 else 0] = False
    return w


def road():
    """The state grid and origin of DESIGN.md §8.20's road request."""
    cam = synth.KITTI
    ctx = capi.Context(cam, max_batch=16, max_local_surfels=1 << 18)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    imgs = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(8)]
    ctx.fuse_stream_resident(list(range(8)), np.stack([g for g, _ in imgs]), np.stack([d for _, d in imgs]),
                             np.stack([synth.pose_stream(t) for t in range(8)]))
    ctx.field_enable(0.2, 64, 20, 128)
    ctx.views_enable(256, 40.0)
    poses = []
    for j in range(256):
        ctx.views_capture(j % 8, j)
        P = np.asarray(synth.pose_stream(j % 8), np.float64).reshape(4, 4).T[:3, :4].reshape(12)   # column-major to [R | t]
        P[3] += 0.35 * (j // 8 % 8) - 1.2
        P[11] += 0.8 * (j // 64)
        poses.append(P)
    ctx.field_enqueue_known((0.0, 1.0, 12.8), 1, list(range(256)), np.array(poses))
    _, origin, _ = ctx.field_wait()
    state, _ = ctx.field_state()
    state, origin = state.copy(), origin.copy()
    ctx.close()
    return state, origin


def cases(rng):
    state, origin = road()
    yield "road", (state, origin, 0.2, -2)
    for n in (320, 1024):
        yield f"obstacles {n}", (floored(obstacles(n, rng)), np.zeros(3, np.int32), 0.1, 3)
    yield "serpentine 256", (floored(serpentine(256)), np.zeros(3, np.int32), 0.1, 3)


def points(origin, voxel, up, terrain):
    """A start and three goals of the terrain's plane (see the module's docstring)."""
    h0, h1 = RT.plane_axes(up)
    info, _, status, _, clear = terrain
    Q, P = int(info["m"][h1]), int(info["m"][h0])
    trav = R.traversable(status, clear, 0.0).reshape(1, Q, P)
    qs, ps = np.nonzero(trav[0])
    if len(qs) == 0:
        raise RuntimeError("no traversable cell")
    i = int(np.argmin(qs + ps))
    cost = R.dijkstra(trav, int(qs[i] * P + ps[i])).reshape(Q, P).astype(np.int64)
    rq, rp = np.nonzero(cost != R.INF)
    far = int(np.argmax(cost[rq, rp]))
    mid = int(np.argmin(np.abs(rq - Q // 2) + np.abs(rp - P // 2)))
    corner = int(np.argmin(rq + (P - rp)))
    cells = [(qs[i], ps[i])] + [(rq[j], rp[j]) for j in (far, mid, corner)]
    v = float(np.float32(voxel))
    pts = []
    for q, p in cells:
        c = [0.0, 0.0, 0.0]
        c[h0], c[h1] = (p + origin[h0] + 0.5) * v, (q + origin[h1] + 0.5) * v
        pts.append(tuple(c))
    return pts[0], pts[1:]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--caps", nargs="+", type=int, default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.lib:
        capi.LIB_PATH = os.path.abspath(a.lib)
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    res = {"card": name, "power_limit": power, "lib": a.lib or "built", "cases": []}
    rng = np.random.default_rng(1)
    for label, (state, origin, voxel, up) in cases(rng):
        nz, ny, nx = state.shape
        terrain = None
        for cap in a.caps:
            ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=1 << 12)
            ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
            ctx.field_enable(voxel, nx, ny, nz)
            ctx.views_enable(1, 1.0)
            ctx.terrain_enable(up)
            ctx.reach_enable(16, 1 << 20, cap)
            ctx.debug_field_load_state(state, origin)
            ctx.field_wait()
            ctx.terrain_enqueue(HEADROOM, MAX_STEP)
            terrain = ctx.terrain_wait()
            if cap == a.caps[0]:
                start, goals = points(origin, voxel, up, terrain)
            g = np.ascontiguousarray(goals, np.float64)
            st3 = (capi.ctypes.c_double * 3)(*start)
            lib, h = ctx.lib, ctx.h
            ctx.reach_enqueue_terrain(start, 0.0, 1, goals, False, True)
            got = ctx.reach_wait()
            exact = None   # another build may use other tiles, so other round counts than the model's
            if not a.lib:
                want = RT.job(terrain, (nx, ny, nz), voxel, start, 0.0, 1, goals, None, 16, 1 << 20, cap)
                exact = all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(got, want))

            def job():
                assert lib.dsm_reach_enqueue_terrain(h, st3, 0.0, 1, g.ctypes.data, len(g), 0, 0) == 0
                assert lib.dsm_reach_wait(h, None, None, None, None) == 0
            for _ in range(3):
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
            for k in prof.key_averages():
                key = next((n for n in KERNELS if n in k.key), "memcpy_dtoh" if "Memcpy DtoH" in k.key else None)
                if key:
                    kern[key] = kern.get(key, 0.0) + k.device_time_total / a.launches
            info = got[0]
            ctx.close()
            r = {"case": label, "grid": [nx, ny, nz], "up": up, "plane": [int(x) for x in terrain[0]["m"]], "max_rounds": cap, "rounds": int(info["rounds"]),
                 "converged": int(info["converged"]), "n_traversable": int(info["n_traversable"]),
                 "n_reached": int(info["n_reached"]), "reached_goals": int((got[1]["status"] == 0).sum()), "bit_exact": exact,
                 "job_ms": spread(ts), "kernels_us_per_job": kern}
            res["cases"].append(r)
            print(json.dumps(r), flush=True)
        # the host alternative: the status and clearance planes to the host, then Dijkstra on the 8-connected graph
        info, _, status, _, clear = terrain
        cells = status.size
        dev = torch.zeros(5 * cells, dtype=torch.uint8, device="cuda")
        host = torch.empty(5 * cells, dtype=torch.uint8).pin_memory()
        copy_ms, dijkstra_ms = [], []
        h0, h1 = RT.plane_axes(up)
        Q, P = int(info["m"][h1]), int(info["m"][h0])
        trav = R.traversable(status, clear, 0.0).reshape(1, Q, P)
        u = int(np.flatnonzero(trav.reshape(-1))[0])
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host.copy_(dev, non_blocking=True)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            R.dijkstra(trav, u)
            t2 = time.perf_counter()
            copy_ms.append((t1 - t0) * 1e3)
            dijkstra_ms.append((t2 - t1) * 1e3)
        r = {"case": label, "host_alternative": {"planes_d2h_ms": spread(copy_ms), "scipy_dijkstra_ms": spread(dijkstra_ms)}}
        res["cases"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        tag = "" if not a.lib else "_" + os.path.splitext(os.path.basename(a.lib))[0]
        with open(os.path.join(a.out, f"measure_reach_terrain{tag}.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
