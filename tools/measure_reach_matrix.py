"""Measure the matrix jobs (dsm_reach_matrix_*, DESIGN.md §8.13) against the paths a planner has without them.

Known fields of tools/measure_field_known.py's scene at 0.2 m for every --grids grid, and the loaded 50 %-random
320x320x40 grid.  Sites: the viewpoints of a reach job from the scene's centre toward the frontier clusters of
frontiers(1), then random traversable voxels, K of them for every --sites K, as voxel centres.  Per K:
  - the matrix job's latency, host clock from dsm_reach_matrix_enqueue to the end of dsm_reach_matrix_wait on an idle
    stream (median, min-max of --reps), its kernels from torch.profiler, n_active_tiles, rounds and converged sites;
  - the same entries from K sequential reach jobs, each started at one site with the other sites' voxel centres as
    goals at approach 0 (how a caller gets them without this job), checked against the matrix;
  - scipy's all-pairs Dijkstra from the K sites on the host copy (oracle/pyoracle_reach.graph), checked against the
    matrix when every site converged; skipped above 2^26 sites x traversable voxels.
Both jobs use --max-rounds.  The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_reach_matrix.py [--sites 16 64 256] [--out DIR]"""
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
from measure_drive import card, kernel_us, spread  # noqa: E402
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
import pyoracle_reach  # noqa: E402

KERNELS = ["k_rm_tiles", "k_rm_slots", "k_rm_sites", "k_rm_init", "k_rm_round", "k_rm_reached", "k_rm_gather", "DeviceScan"]


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


def loader(grid, max_sites, max_rounds):
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(4096, 1 << 20)
    ctx.reach_enable(max(max_sites, 4096), 1 << 18, max_rounds)
    tiles = int(np.prod([(n + 7) // 8 for n in grid]))
    ctx.reach_matrix_enable(max_sites, min(tiles, (1 << 34) // (4096 * max_sites)), max_rounds)   # within 2^34 B of costs
    return ctx


def centres(u, origin, shape_zyx):
    nz, ny, nx = shape_zyx
    c = np.stack([u % nx, u // nx % ny, u // (nx * ny)], 1).astype(np.float64)
    return (c + np.asarray(origin, np.float64) + 0.5) * float(np.float32(VOXEL))


def measure(state, origin, start, ks, max_rounds, reps, launches, what, rng):
    grid = state.shape[::-1]
    ctx = loader(grid, max(ks), max_rounds)
    ctx.debug_field_load_state(state, origin)
    dist = ctx.field_wait()[0]
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    ctx.reach_enqueue(start, VOXEL, 2, None, True, False)
    _, targets, _, _ = ctx.reach_wait()
    vp = np.unique(targets["viewpoint"][targets["status"] == 0]).astype(np.int64)
    trav = pyoracle_reach.traversable(state, dist, VOXEL)
    idx = np.flatnonzero(trav.reshape(-1))
    rest = rng.permutation(np.setdiff1d(idx, vp))
    order = np.concatenate([vp, rest])
    g = pyoracle_reach.graph(trav)
    r = {"what": what, "grid": grid, "max_rounds": max_rounds, "n_traversable": int(trav.sum()), "viewpoints": int(len(vp)), "by_sites": []}
    for k in ks:
        u = order[:k]
        pts = centres(u, origin, state.shape)

        def matrix():
            ctx.reach_matrix_enqueue(pts, VOXEL, 0)
            return ctx.reach_matrix_wait()

        def sequential():
            out = []
            for i in range(k):
                ctx.reach_enqueue(pts[i], VOXEL, 0, pts, False, False)
                out.append(ctx.reach_wait())
            return out
        info, sites, M = matrix()
        assert (sites["voxel"] == u).all(), f"{what}: a site did not snap to itself"
        seq = sequential()
        S = np.stack([t["cost"] for _, t, _, _ in seq])
        assert S.tobytes() == M.tobytes(), f"{what} K={k}: sequential reach jobs and the matrix differ"
        e = {"sites": k, "n_active_tiles": int(info["n_active_tiles"]), "rounds": int(info["rounds"]),
             "converged_sites": int(sites["converged"].sum()), "matrix_ms": timed(matrix, reps, ctx),
             "sequential_ms": timed(sequential, max(1, reps // 4), ctx)}
        per = kernel_us(lambda: [matrix() for _ in range(launches)], KERNELS)
        e["kernels_us"] = {n: sum(v) / launches for n, v in per.items() if v}
        e["round_launches"] = len(per["k_rm_round"]) // launches
        if k * r["n_traversable"] > 1 << 26:   # minutes of host time: not measured
            r["by_sites"].append(e)
            print(json.dumps(e), flush=True)
            continue
        t0 = time.perf_counter()
        d = csgraph.dijkstra(g, directed=False, indices=u)[:, u]
        e["scipy_all_pairs_ms"] = (time.perf_counter() - t0) * 1e3
        if sites["converged"].all():
            assert M.tobytes() == np.where(np.isfinite(d), d, pyoracle_reach.INF).astype(np.uint32).tobytes(), f"{what} K={k}: Dijkstra"
        r["by_sites"].append(e)
        print(json.dumps(e), flush=True)
    ctx.close()
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--sites", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--max-rounds", type=int, default=256)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--skip-random", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "known": [], "loaded": []}
    rng = np.random.default_rng(3)
    for gs in a.grids:
        grid = tuple(int(x) for x in gs.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)
        ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses, host_copy=True)
        origin = ctx.field_wait()[1]
        state = ctx.field_state()[0].copy()
        ctx.close()
        res["known"].append(measure(state, origin, c, a.sites, a.max_rounds, a.reps, a.launches, f"{gs} scene", rng))
    if not a.skip_random:
        grid, o = (320, 320, 40), (-160, -160, -5)
        st = rng.choice([1, 2], size=grid[::-1]).astype(np.uint8)
        start = ((o[0] + grid[0] / 2) * VOXEL, (o[1] + grid[1] / 2) * VOXEL, (o[2] + grid[2] / 2) * VOXEL)
        res["loaded"].append(measure(st, o, start, a.sites, a.max_rounds, a.reps, a.launches, "random 50 % free", rng))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_reach_matrix.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
