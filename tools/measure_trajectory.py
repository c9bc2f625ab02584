"""Measure the trajectory job (dsm_trajectory_*, DESIGN.md §8.17) against the same optimiser driven on the host.

On tools/measure_field.py's map (a store of --store surfels over the box, voxel 0.1 m) with the signed grid, for 1, 64
and 4096 trajectories of 16 to 64 control points at --iters iterations:
1. the device job: host clock from dsm_trajectory_enqueue to the end of dsm_trajectory_wait on an idle stream (--reps
   runs), and k_trajectory's kernel time from torch.profiler in a run of its own;
2. the host loop: oracle/pyoracle_trajectory's optimiser with every cost evaluation's field samples taken by a signed
   dsm_field_query_enqueue / _wait round trip, on the first --host trajectories (per trajectory, and times n);
3. the numpy model on the same trajectories (per trajectory, and times n).
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_trajectory.py [--counts 1 64 4096] [--out DIR]"""
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
from measure_drive import card, spread  # noqa: E402
from measure_field import VOXEL, stored_context  # noqa: E402
import pyoracle_trajectory as tj  # noqa: E402

GRID = (200, 200, 60)


def trajectories(rng, n):
    ext = np.array(GRID, np.float64) * VOXEL * 0.8
    lens = rng.integers(16, 65, n)
    pts = []
    for N in lens:
        a, b = (rng.random(3) - 0.5) * ext, (rng.random(3) - 0.5) * ext
        pts.append(a + np.linspace(0, 1, N)[:, None] * (b - a) + rng.standard_normal((N, 3)) * 0.1)
    return np.concatenate(pts), np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), rng.uniform(0.3, 1.0, n)


def query_sampler(ctx):
    """The optimiser's field samples through one signed point-query round trip each."""
    def sampler(p):
        ctx.field_query_enqueue(p, signed=True)
        s = ctx.field_query_wait()[0]
        return ~np.isnan(s["dist"]), s["dist"].astype(np.float64), np.stack([s["gx"], s["gy"], s["gz"]], 1).astype(np.float64)
    return sampler


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--counts", nargs="+", type=int, default=[1, 64, 4096])
    ap.add_argument("--store", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    ctx = stored_context(a.store, GRID)
    ctx.field_signed_enable()
    ctx.field_query_enable(64, 1, 2)
    ctx.trajectory_enable(max(a.counts), 64 * max(a.counts), 8)
    ctx.field_enqueue((0.0, 0.0, 0.0), 5)
    _, origin, _ = ctx.field_wait()
    sdist = ctx.field_signed()
    p = tj.params(1, 10, 1, margin=0.5, v_max=2.0, a_max=4.0, g_tol=0.0, max_iter=a.iters, memory=8, max_ls=16, samples=8)
    res = {"card": name, "power_limit": power, "store_surfels": a.store, "grid": GRID, "params": p, "runs": []}
    rng = np.random.default_rng(1)
    for n in a.counts:
        pts, ofs, dt = trajectories(rng, n)
        r = {"trajectories": n, "points": int(ofs[-1])}
        for _ in range(2):   # warm
            ctx.trajectory_enqueue(pts, ofs, dt, p)
            ctx.trajectory_wait()
        ts = []
        for _ in range(a.reps):
            ctx.sync()
            t0 = time.perf_counter()
            ctx.trajectory_enqueue(pts, ofs, dt, p)
            _, rec, _ = ctx.trajectory_wait()
            ts.append((time.perf_counter() - t0) * 1e3)
        r["device_ms"] = spread(ts)
        r["iterations"] = spread(rec["iterations"].tolist())
        r["status"] = np.bincount(rec["status"], minlength=4).tolist()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                ctx.trajectory_enqueue(pts, ofs, dt, p)
                ctx.trajectory_wait()
            torch.cuda.synchronize()
        rows = [k for k in prof.key_averages() if "k_trajectory" in k.key]
        if sum(k.count for k in rows) != a.reps:
            raise RuntimeError("profiler did not see one k_trajectory per job")
        r["kernel_ms"] = sum(k.device_time_total for k in rows) / a.reps / 1e3
        m = min(n, a.host)
        sub = ofs[:m + 1]
        for key, sampler in (("host_loop", query_sampler(ctx)), ("model", tj.grid_sampler(sdist, origin, VOXEL))):
            t0 = time.perf_counter()
            for j in range(m):
                tj.optimise(pts[sub[j]:sub[j + 1]], dt[j], p, sampler, VOXEL)
            per = (time.perf_counter() - t0) * 1e3 / m
            r[key] = {"measured_trajectories": m, "ms_per_trajectory": per, "ms_times_n": per * n}
        res["runs"].append(r)
        print(json.dumps(r), flush=True)
    ctx.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_trajectory.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
