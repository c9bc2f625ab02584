"""Measure the tour jobs (dsm_tour_*, DESIGN.md §8.14) against running the same search on the host.

  - Latency: host clock from dsm_tour_enqueue to the end of dsm_tour_wait on an idle stream (median, min-max of
    --reps) for every n in --sites against every n_starts in --starts, on stretched metric matrices (Euclidean distances
    between random points, each entry times a factor in [1, 1.3]) with max_passes the largest the work bound allows, at
    most --max-passes; with the passes the starts took and how many converged.  The n_starts = 1 jobs are checked bit
    for bit against oracle/pyoracle_tour, whose time per start is the figure for running without this job (LKH, the
    solver FUEL uses, is not available here).
  - The job's kernels from torch.profiler.
  - Quality: the best start's gap to the Held-Karp optimum over --hk-instances instances at n = 8 and 13, open and
    closed; and the best of 256 starts against start 0 (nearest neighbour and its local search) on the matrices of
    matrix jobs over tools/measure_reach_matrix.py's scene field at 0.2 m.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_tour.py [--sites 16 64 256 1024] [--starts 1 32 256] [--out DIR]"""
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
from measure_drive import card, kernel_us, spread  # noqa: E402
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
from measure_reach_matrix import centres, loader  # noqa: E402
import pyoracle_reach  # noqa: E402
import pyoracle_tour as TM  # noqa: E402

KERNELS = ["k_tour_search", "k_tour_best"]


def metric(n, rng):
    p = rng.uniform(0, 100, (n, 2))
    d = np.linalg.norm(p[:, None] - p[None], axis=-1)
    return np.round(d * rng.uniform(1.0, 1.3, (n, n)) * 10).astype(np.uint32)


def held_karp(W):
    """The least tour cost from site 0 over all n sites of the int64 weights W (the open rule already in W)."""
    n = len(W)
    k = n - 1
    big = np.iinfo(np.int64).max // 4
    dp = np.full((1 << k, k), big, np.int64)
    dp[1 << np.arange(k), np.arange(k)] = W[0, 1:]
    Wr = W[1:, 1:]
    for mask in range(1, 1 << k):
        ends = np.flatnonzero((mask >> np.arange(k)) & 1)
        if len(ends) < 2:
            continue
        for j in ends:
            prev = mask ^ (1 << int(j))
            dp[mask, j] = (dp[prev, ends] + Wr[ends, j]).min()
    return int((dp[(1 << k) - 1] + W[1:, 0]).min())


def timed(fn, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def latency(ctx, ns, ks, cap, reps, launches, rng):
    out = []
    for n in ns:
        M = metric(n, rng)
        for k in ks:
            passes = min(cap, TM.MAX_WORK // (k * n * n))

            def run():
                ctx.tour_enqueue(M, 0, k, passes, 1)
                return ctx.tour_wait()
            info, starts, order = run()
            e = {"sites": n, "starts": k, "max_passes": passes, "job_ms": timed(run, reps),
                 "passes": spread(starts["passes"].tolist()), "converged": int(starts["converged"].sum()),
                 "best_cost": int(info["best_cost"]), "start0_cost": int(starts["cost"][0])}
            per = kernel_us(lambda: [run() for _ in range(launches)], KERNELS)
            e["kernels_us"] = {name: sum(v) / launches for name, v in per.items() if v}
            if k == 1:
                t0 = time.perf_counter()
                want = TM.tour(M, 0, 1, passes, 1)
                e["host_model_ms_per_start"] = (time.perf_counter() - t0) * 1e3
                assert all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip((info, starts, order), want)), f"n={n}: model"
            out.append(e)
            print(json.dumps(e), flush=True)
    return out


def held_karp_gap(ctx, instances, rng):
    out = []
    for n in (8, 13):
        for open_ in (0, 1):
            gaps, optimal = [], 0
            for _ in range(instances):
                M = metric(n, rng)
                ctx.tour_enqueue(M, open_, 32, 64, 3)
                info = ctx.tour_wait()[0]
                hk = held_karp(TM.weights(M, open_))
                gaps.append((int(info["best_cost"]) - hk) / max(hk, 1))
                optimal += int(info["best_cost"]) == hk
            e = {"sites": n, "open": open_, "instances": instances, "starts": 32, "optimal": optimal,
                 "gap_mean": float(np.mean(gaps)), "gap_max": float(np.max(gaps))}
            out.append(e)
            print(json.dumps(e), flush=True)
    return out


def scene_matrices(ks, rng):
    """Best of 256 starts against start 0 on matrix jobs over the scene's known field at 320x320x40."""
    grid = (320, 320, 40)
    sctx, poses, views, c = scene()
    sctx.field_enable(VOXEL, *grid)
    sctx.views_enable(MAX_VIEWS, MAX_RANGE)
    for j in range(MAX_VIEWS):
        sctx.views_capture(j % 8, j)
    sctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses, host_copy=True)
    origin = sctx.field_wait()[1]
    state = sctx.field_state()[0].copy()
    sctx.close()
    ctx = loader(grid, max(ks), 256)
    ctx.tour_enable(max(ks), 256)
    ctx.debug_field_load_state(state, origin)
    dist = ctx.field_wait()[0]
    idx = np.flatnonzero(pyoracle_reach.traversable(state, dist, VOXEL).reshape(-1))
    out = []
    for k in ks:
        pts = centres(np.concatenate([[idx[len(idx) // 2]], rng.choice(idx, k - 1, replace=False)]), origin, state.shape)
        ctx.reach_matrix_enqueue(pts, VOXEL, 0)
        M = ctx.reach_matrix_wait()[2]
        for open_ in (0, 1):
            passes = min(4096, TM.MAX_WORK // (256 * k * k))
            ctx.tour_enqueue(M, open_, 256, passes, 5)
            info, starts, _ = ctx.tour_wait()
            e = {"sites": k, "open": open_, "n_included": int(info["n_included"]), "max_passes": passes,
                 "best_cost": int(info["best_cost"]), "start0_cost": int(starts["cost"][0]),
                 "best_over_start0": int(info["best_cost"]) / max(int(starts["cost"][0]), 1),
                 "passes": spread(starts["passes"].tolist()), "converged": int(starts["converged"].sum())}
            out.append(e)
            print(json.dumps(e), flush=True)
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sites", type=int, nargs="+", default=[16, 64, 256, 1024])
    ap.add_argument("--starts", type=int, nargs="+", default=[1, 32, 256])
    ap.add_argument("--max-passes", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--launches", type=int, default=2)
    ap.add_argument("--hk-instances", type=int, default=50)
    ap.add_argument("--scene-sites", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rng = np.random.default_rng(7)
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.tour_enable(max(a.sites), max(a.starts + [32]))
    res = {"card": name, "power_limit": power, "latency": latency(ctx, a.sites, a.starts, a.max_passes, a.reps, a.launches, rng),
           "held_karp": held_karp_gap(ctx, a.hk_instances, rng)}
    ctx.close()
    res["scene"] = scene_matrices(a.scene_sites, rng)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_tour.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
