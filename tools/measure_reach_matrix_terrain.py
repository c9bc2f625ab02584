"""Measure the terrain matrix job (dsm_reach_matrix_enqueue_terrain, DESIGN.md §8.22) against the two paths a ground
planner takes without it.

Cases, each a terrain job (headroom 5, max step 1) on a loaded known field, then a matrix over K sites of its plane (the
centres of K traversable cells drawn at random, seeded):
  road        the synthetic road request of DESIGN.md §8.20 (tools/measure_reach_terrain.road), up = -2;
  obstacles   320 x 320 and 1024 x 1024 z-up planes: an occupied floor with 8 % of the columns unobserved and long walls
              with one gap each (tools/measure_reach_terrain.obstacles), so that nearly every flat tile is active.
Per case and per K in --sites (max_rounds 4096, max_tiles the plane's flat tile count):
1. The matrix job: host clock from dsm_reach_matrix_enqueue_terrain to the end of dsm_reach_matrix_wait, median and range
   of --reps, and the per-kernel device times of torch.profiler (CUDA activities, --launches jobs).
2. K sequential terrain reach jobs (dsm_reach_enqueue_terrain with the cost grid copied to the host), one per site, read
   at the sites: the same entries, checked equal; one pass timed.
3. The host alternative: the status and clearance planes (5 B per cell) copied device to host (pinned, torch), then
   scipy's Dijkstra on the 8-connected 10/14 graph from the sites: checked equal.  On planes above --host-cells cells
   only the first --host-rows sites run, and the time is reported per row.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_reach_matrix_terrain.py [--sites 16 64 256] [--reps 10] [--out DIR]"""
import argparse
import json
import os
import sys
import time

import numpy as np
from scipy.sparse import csgraph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import card, spread  # noqa: E402
from measure_reach_terrain import HEADROOM, MAX_STEP, floored, obstacles, road  # noqa: E402
import pyoracle_reach as R  # noqa: E402
import pyoracle_reach_matrix_terrain as RMT  # noqa: E402
import pyoracle_reach_terrain as RT  # noqa: E402

KERNELS = ("k_rm_round", "k_rm_init", "k_rm_tiles", "k_rm_sites", "k_rm_slots", "k_rm_reached", "k_rm_gather", "DeviceScan")
ROUNDS = 4096


def cases(rng):
    state, origin = road()
    yield "road", (state, origin, 0.2, -2)
    for n in (320, 1024):
        yield f"obstacles {n}", (floored(obstacles(n, rng)), np.zeros(3, np.int32), 0.1, 3)


def sites(terrain, voxel, k, rng):
    """The world centres of k traversable cells drawn at random, and those cells."""
    trav = RMT.plane(terrain, 0.0)[0]
    up = int(terrain[0]["up"])
    h0, h1 = RT.plane_axes(up)
    P = trav.shape[1]
    cells = rng.choice(np.flatnonzero(trav), size=k, replace=False)
    v = float(np.float32(voxel))
    pts = np.zeros((k, 3))
    pts[:, h0] = (cells % P + int(terrain[0]["origin"][h0]) + 0.5) * v
    pts[:, h1] = (cells // P + int(terrain[0]["origin"][h1]) + 0.5) * v
    return pts, cells


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sites", nargs="+", type=int, default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--host-cells", type=int, default=200_000)
    ap.add_argument("--host-rows", type=int, default=8)
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
        h0, h1 = RT.plane_axes(up)
        n0, n1 = state.shape[::-1][h0], state.shape[::-1][h1]
        flat_tiles = ((n0 + 31) // 32) * ((n1 + 15) // 16)
        ctx.reach_matrix_enable(max(a.sites), flat_tiles, ROUNDS)
        ctx.reach_enable(1, 1, ROUNDS)
        ctx.debug_field_load_state(state, origin)
        ctx.field_wait()
        ctx.terrain_enqueue(HEADROOM, MAX_STEP)
        terrain = ctx.terrain_wait()
        trav = RMT.plane(terrain, 0.0)[0]
        lib, h = ctx.lib, ctx.h
        for k in a.sites:
            if k > trav.sum():
                continue
            pts, cells = sites(terrain, voxel, k, rng)
            ctx.reach_matrix_enqueue_terrain(pts, 0.0, 0)
            info, srec, M = ctx.reach_matrix_wait()

            def job():
                assert lib.dsm_reach_matrix_enqueue_terrain(h, pts.ctypes.data, k, 0.0, 0) == 0
                assert lib.dsm_reach_matrix_wait(h, None, None, None) == 0
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
                key = next((n for n in KERNELS if n in e.key), "memcpy" if "Memcpy" in e.key else "memset" if "Memset" in e.key else None)
                if key:
                    kern[key] = kern.get(key, 0.0) + e.device_time_total / a.launches
            # K terrain reach jobs, one per site, read at the sites
            ctx.sync()
            t0 = time.perf_counter()
            rows = []
            for p in pts:
                ctx.reach_enqueue_terrain(tuple(p), 0.0, 0, None, False, True)
                rows.append(ctx.reach_wait()[3].reshape(-1)[cells])
            k_jobs_ms = (time.perf_counter() - t0) * 1e3
            k_jobs_equal = bool(np.array_equal(np.stack(rows), M))
            # the host alternative
            dev = torch.zeros(5 * trav.size, dtype=torch.uint8, device="cuda")
            host = torch.empty(5 * trav.size, dtype=torch.uint8).pin_memory()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host.copy_(dev, non_blocking=True)
            torch.cuda.synchronize()
            copy_ms = (time.perf_counter() - t0) * 1e3
            n_rows = k if trav.size <= a.host_cells else min(k, a.host_rows)
            t0 = time.perf_counter()
            d = csgraph.dijkstra(R.graph(trav[None]), directed=False, indices=cells[:n_rows])[:, cells]
            dijkstra_ms = (time.perf_counter() - t0) * 1e3
            host_equal = bool(np.array_equal(np.where(np.isfinite(d), d, R.INF).astype(np.uint32), M[:n_rows]))
            r = {"case": label, "grid": [nx, ny, nz], "up": up, "plane": [n0, n1], "flat_tiles": flat_tiles, "sites": k,
                 "n_active_tiles": int(info["n_active_tiles"]), "rounds": int(info["rounds"]), "status": int(info["status"]),
                 "converged": bool((srec["converged"] == 1).all()), "matrix_ms": spread(ts), "kernels_us_per_job": kern,
                 "k_reach_jobs_ms": k_jobs_ms, "k_reach_jobs_equal": k_jobs_equal,
                 "host": {"planes_d2h_ms": copy_ms, "scipy_rows": n_rows, "scipy_dijkstra_ms": dijkstra_ms,
                          "scipy_ms_per_row": dijkstra_ms / n_rows, "equal": host_equal}}
            res["cases"].append(r)
            print(json.dumps(r), flush=True)
        ctx.close()
    print(json.dumps({"card": name, "power_limit": power}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_reach_matrix_terrain.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
