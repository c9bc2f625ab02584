"""Measure the terrain job (dsm_terrain_*, DESIGN.md §8.20) against the path a ground planner takes without it.

The scene field of tools/measure_field_known.py (eight fused synthetic frames in 256 captured views, a known request at
0.2 m centred on frame 4's camera) is built once per --grids grid and its state grid read back.  It is then loaded
(dsm_debug_field_load_state) into a context per case: up = +3 on the grid as built and up = -2 on the grid with its y
and z axes swapped, so that both coalesced walks are timed on the same voxels, and up = -2 on the grid as built, the
scene's own up axis (y down), the case a KITTI-frame planner runs.  Per case, at --headroom and --max-step:
1. Latency: host clock from dsm_terrain_enqueue to the end of dsm_terrain_wait (through the C calls), median of --reps
   on an idle stream.
2. Per-kernel device times from torch.profiler (CUDA activities, --launches jobs): k_terrain_support, k_terrain_step,
   the three EDT passes and the result's D2H copy.
3. Today's path: the state grid copied device to host (pinned, torch), then oracle/pyoracle_terrain on it in numpy.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_terrain.py [--grids 320x320x40 512x512x64] [--reps 50] [--out DIR]"""
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
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
import pyoracle_terrain as TR  # noqa: E402

KERNELS = ("k_terrain_support", "k_terrain_step", "k_field_rows", "k_field_lines")


def scene_state(grid):
    """The state grid [nz][ny][nx] and origin of the scene's known request on `grid` with every view."""
    ctx, poses, views, c = scene()
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(MAX_VIEWS, MAX_RANGE)
    for j in range(MAX_VIEWS):
        ctx.views_capture(j % 8, j)
    ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses)
    _, origin, _ = ctx.field_wait()
    state, _ = ctx.field_state()
    state, origin = state.copy(), origin.copy()
    ctx.close()
    return state, origin


def loaded(state, origin, up):
    nz, ny, nx = state.shape
    ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, nx, ny, nz)
    ctx.views_enable(1, 1.0)
    ctx.terrain_enable(up)
    ctx.debug_field_load_state(state, origin)
    ctx.field_wait()
    return ctx


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["320x320x40", "512x512x64"])
    ap.add_argument("--headroom", type=int, default=5)
    ap.add_argument("--max-step", type=int, default=1)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "headroom": a.headroom, "max_step": a.max_step, "cases": []}
    for g in a.grids:
        grid = tuple(int(x) for x in g.split("x"))
        state, origin = scene_state(grid)
        swapped = np.ascontiguousarray(state.transpose(1, 0, 2))
        for up, st, org in ((3, state, origin), (-2, swapped, origin[[0, 2, 1]]), (-2, state, origin)):
            ctx = loaded(st, org, up)
            lib, h = ctx.lib, ctx.h
            want = TR.job(st, org, VOXEL, up, a.headroom, a.max_step)
            ctx.terrain_enqueue(a.headroom, a.max_step)
            got = ctx.terrain_wait()
            exact = all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(got, want))

            def job():
                assert lib.dsm_terrain_enqueue(h, a.headroom, a.max_step) == 0
                assert lib.dsm_terrain_wait(h, None, None, None, None, None) == 0
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
            ctx.close()
            # today's path: the state grid to the host, then the model in numpy
            dev = torch.from_numpy(st).cuda()
            host = torch.empty(st.shape, dtype=torch.uint8).pin_memory()
            copy_ms, model_ms = [], []
            for _ in range(max(3, a.reps // 10)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                host.copy_(dev, non_blocking=True)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                TR.job(host.numpy(), org, VOXEL, up, a.headroom, a.max_step)
                t2 = time.perf_counter()
                copy_ms.append((t1 - t0) * 1e3)
                model_ms.append((t2 - t1) * 1e3)
            info = got[0]
            r = {"grid": [int(x) for x in st.shape[::-1]], "up": up, "bit_exact": exact, "n_support": int(info["n_support"]),
                 "n_traversable": int(info["n_traversable"]), "n_blocked": int(info["n_blocked"]),
                 "result_bytes": int(8 * np.prod(info["m"]) + 32), "job_ms": spread(ts), "kernels_us_per_job": kern,
                 "state_d2h_ms": spread(copy_ms), "numpy_model_ms": spread(model_ms)}
            res["cases"].append(r)
            print(json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_terrain.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
