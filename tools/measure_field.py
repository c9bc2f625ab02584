"""Measure the distance field of the resident map (dsm_field_*, DESIGN.md §8.7).

1. Kernels (torch.profiler, CUDA activities, --launches requests) for every --grids grid and --stores store size: a
   context whose store holds N surfels spread uniformly over the grid's box (pool empty), voxel 0.1 m, centre in the
   box.  Per request: k_field_mark, k_field_rows, the y and z envelope passes, the memset and the D2H copy.  Model bytes:
   mark 44 B per surfel read; each EDT pass 4 B read and 4 B written per voxel; share of the data sheet's 3.35 TB/s.
2. Latency: host clock from dsm_field_enqueue to the end of dsm_field_wait, D2H copy included, on an idle stream.
3. Host baseline: what a planner does today with the same map: the two clouds to the host (dsm_pool_export_cloud +
   dsm_inactive_export_cloud), voxelised with numpy, scipy.ndimage.distance_transform_edt on the host CPU.
4. The node drive of tools/measure_node.py (1226x370, --frames frames) through dsm::SurfelMapNode
   (tools/measure_field.cpp), modes alternating on fresh nodes, --rounds rounds: a no field; f the field of frame t-1
   taken at the start of frame t; g the field taken right after every fuse.  Grid --node-grid at --node-voxel.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_field.py [--frames 320] [--rounds 3] [--out DIR]"""
import argparse
import ctypes
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import SMALL, build_harness, card, images, messages, run_harness, spread, write_drive  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
VOXEL = 0.1
KERNELS = {"mark": "k_field_mark", "rows": "k_field_rows", "y_pass": "k_field_lines<false>", "z_pass": "k_field_lines<true>"}


def node_drive(n_frames, rounds, grid, voxel):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_harness(tmp, "measure_field")
        ff, fs = write_drive(tmp, images(), messages(n_frames))
        times = {m: [] for m in "afg"}
        last = {}
        for _ in range(rounds):
            for m in "afg":
                last[m] = run_harness(exe, ff, fs, [m, voxel, *grid])
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "voxel": voxel, "store_surfels": last["a"]["store_surfels"],
            "pool_surfels": last["a"]["pool_surfels"], "mean_occupied_voxels": last["f"]["occupied"] / max(last["f"]["fields"], 1),
            "ms_per_frame": {m: spread(times[m]) for m in "afg"}}


def stored_context(n, grid):
    """A context whose store holds n surfels as one segment, spread uniformly over the box of `grid` at VOXEL around the
    origin; pool empty; the field enabled."""
    from densesurfelmapping_b200 import capi
    ctx = capi.Context(SMALL, max_batch=1, max_local_surfels=max(n, 1 << 16))
    rng = np.random.default_rng(7)
    s = np.zeros(n, SURFEL_DTYPE)
    ext = np.array(grid, np.float64) * VOXEL
    p = (rng.random((n, 3)) - 0.5) * ext
    s["px"], s["py"], s["pz"] = p[:, 0], p[:, 1], p[:, 2]
    s["nz"], s["size"], s["weight"], s["update_times"], s["last_update"], s["color"] = 1.0, 0.1, 1.0, 7, 0, 100.0
    ctx.pool_upload(s)
    ctx.inactive_reserve(n)
    assert ctx.inactive_retire(0) == n
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    return ctx


def kernels(ctx, n, grid, launches):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib, h = ctx.lib, ctx.h
    c = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for _ in range(5):
        assert lib.dsm_field_enqueue(h, c, 5) == 0 and lib.dsm_field_wait(h, None, None, None) == 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            assert lib.dsm_field_enqueue(h, c, 5) == 0
            assert lib.dsm_field_wait(h, None, None, None) == 0
        torch.cuda.synchronize()
    voxels = grid[0] * grid[1] * grid[2]
    out = {}
    for name, key in KERNELS.items():
        rows = [k for k in prof.key_averages() if key in k.key]
        count = sum(k.count for k in rows)
        if count != launches:
            raise RuntimeError(f"profiler saw {count} launches of {key}, expected {launches}")
        us = sum(k.device_time_total for k in rows) / count
        nbytes = 44 * n if name == "mark" else 8 * voxels
        out[name] = {"us": us, "model_bytes": nbytes, "share_of_3.35TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}
    for name, key in (("memset", "Memset"), ("d2h_copy", "Memcpy DtoH")):
        rows = [k for k in prof.key_averages() if key in k.key]
        count = sum(k.count for k in rows)
        us = sum(k.device_time_total for k in rows) / max(launches, 1)
        out[name] = {"us_per_request": us, "ops": count}
    out["d2h_copy"]["bytes"] = 4 * voxels
    out["kernels_us"] = sum(out[k]["us"] for k in KERNELS)
    return out


def latency(ctx, reps):
    lib, h = ctx.lib, ctx.h
    c = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        assert lib.dsm_field_enqueue(h, c, 5) == 0
        assert lib.dsm_field_wait(h, None, None, None) == 0
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def host_baseline(ctx, grid, reps):
    """The planner of today: both clouds to the host, voxelised, scipy's EDT (distances only), one CPU core."""
    from scipy import ndimage
    import pyoracle_field
    ts, edt = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        pts = np.concatenate([ctx.pool_export_cloud(5).view(np.float32).reshape(-1, 4)[:, :3],
                              ctx.inactive_export_cloud().view(np.float32).reshape(-1, 4)[:, :3]])
        o = pyoracle_field.origin([0.0, 0.0, 0.0], VOXEL, grid)
        occ = pyoracle_field.occupancy(pts, VOXEL, grid, o)
        t1 = time.perf_counter()
        d = ndimage.distance_transform_edt(~occ) * VOXEL
        t2 = time.perf_counter()
        ts.append((t2 - t0) * 1e3)
        edt.append((t2 - t1) * 1e3)
        assert d.shape == occ.shape
    return {"total_ms": spread(ts), "edt_ms": spread(edt)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--stores", type=int, nargs="+", default=[46700, 1 << 20, 1 << 22])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--node-grid", default="320x320x40")
    ap.add_argument("--node-voxel", type=float, default=0.2)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    grids = [tuple(int(x) for x in g.split("x")) for g in a.grids]
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "fields": []}
    for g in grids:
        for n in a.stores:
            ctx = stored_context(n, g)
            r = {"grid": g, "store_surfels": n, "kernels": kernels(ctx, n, g, a.launches), "latency_ms": latency(ctx, 50)}
            if n == 1 << 20:
                r["host_baseline"] = host_baseline(ctx, g, a.host_reps)
            ctx.close()
            res["fields"].append(r)
            print(json.dumps(r), flush=True)
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, tuple(int(x) for x in a.node_grid.split("x")), a.node_voxel)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_field.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
