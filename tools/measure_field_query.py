"""Measure the planner queries against the resident distance field (dsm_field_query_*, DESIGN.md §8.8).

On a 320x320x40 field at 0.2 m over a store of 1 Mi surfels spread uniformly over the grid's box (pool empty), built
with dsm_field_enqueue_resident:
1. Latency: host clock from dsm_field_query_enqueue to the end of dsm_field_query_wait on an idle stream, for 1 Ki,
   64 Ki and 1 Mi random points in the box, and for 1 Ki and 4 Ki trajectories of 32 waypoints (a random walk in the
   box) at step = v / 2.
2. Kernels (torch.profiler, CUDA activities, --launches queries per case): k_field_query and k_field_clearance, with the
   H2D and D2H copies.  Model bytes: a point reads 24 B and writes 16 B, and gathers 8 corners of 4 B; a trajectory
   sample gathers 8 corners of 4 B (its waypoints and segment starts are amortised).  Share of the data sheet's
   3.35 TB/s; the gathers mostly hit L2 (the grid is 16 MB), so the share is an upper-bound model, not HBM traffic.
3. Host baseline: the same queries answered by numpy (oracle/pyoracle_field_query.py) on the host copy of the grid,
   which a planner has today after dsm_field_wait.  The copy's own time is not included.
4. The node drive of tools/measure_node.py (1226x370, --frames frames) through dsm::SurfelMapNode
   (tools/measure_field_query.cpp), modes alternating on fresh nodes, --rounds rounds: h a host-copy field read after
   every fuse; q a resident field plus one 4 Ki-trajectory clearance after every fuse.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_field_query.py [--frames 320] [--rounds 3] [--out DIR]"""
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
GRID, VOXEL, STORE = (320, 320, 40), 0.2, 1 << 20
POINTS = [1 << 10, 1 << 16, 1 << 20]
TRAJECTORIES = [1 << 10, 1 << 12]
PER_TRAJ = 32


def node_drive(n_frames, rounds, grid, voxel):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_harness(tmp, "measure_field_query")
        ff, fs = write_drive(tmp, images(), messages(n_frames))
        times = {m: [] for m in "hq"}
        last = {}
        for _ in range(rounds):
            for m in "hq":
                last[m] = run_harness(exe, ff, fs, [m, voxel, *grid])
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "voxel": voxel, "hits_per_frame": last["q"]["hits"] / max(n_frames, 1),
            "ms_per_frame": {m: spread(times[m]) for m in "hq"}}


def field_context():
    """A context whose store holds STORE surfels spread uniformly over the grid's box around the origin; pool empty; a
    resident field centred on the origin, and its host copy (dist, origin)."""
    from densesurfelmapping_b200 import capi
    ctx = capi.Context(SMALL, max_batch=1, max_local_surfels=STORE)
    rng = np.random.default_rng(7)
    s = np.zeros(STORE, SURFEL_DTYPE)
    p = (rng.random((STORE, 3)) - 0.5) * np.array(GRID, np.float64) * VOXEL
    s["px"], s["py"], s["pz"] = p[:, 0], p[:, 1], p[:, 2]
    s["nz"], s["size"], s["weight"], s["update_times"], s["last_update"], s["color"] = 1.0, 0.1, 1.0, 7, 0, 100.0
    ctx.pool_upload(s)
    ctx.inactive_reserve(STORE)
    assert ctx.inactive_retire(0) == STORE
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *GRID)
    ctx.field_query_enable(max(POINTS), max(TRAJECTORIES), max(TRAJECTORIES) * PER_TRAJ)
    ctx.field_enqueue([0.0, 0.0, 0.0], 5)
    host = ctx.field_wait()
    ctx.field_enqueue([0.0, 0.0, 0.0], 5, host_copy=False)
    ctx.field_wait()
    return ctx, host


def cases(origin):
    rng = np.random.default_rng(3)
    o, n3 = origin.astype(np.float64), np.array(GRID, np.float64)
    v = float(np.float32(VOXEL))
    out = []
    for n in POINTS:
        out.append((f"points_{n}", (o + rng.random((n, 3)) * (n3 - 1) + 0.5) * v, None, None, n))
    for n in TRAJECTORIES:
        start = o + 4 + rng.random((n, 1, 3)) * (n3 - 8)
        wp = (start + np.cumsum(rng.uniform(-1.5, 1.5, (n, PER_TRAJ, 3)), 1)) * v
        out.append((f"trajectories_{n}", None, wp.reshape(-1, 3), np.arange(n + 1, dtype=np.int32) * PER_TRAJ, n))
    return out


def raw_args(pts, wp, ofs):
    """Prepared ctypes arguments of one dsm_field_query_enqueue, so that the timed window holds the library call only."""
    keep = []
    p = w = o = None
    if pts is not None:
        keep.append(np.ascontiguousarray(pts, np.float64))
        p = keep[-1].ctypes.data
    if wp is not None:
        keep += [np.ascontiguousarray(wp, np.float64), np.ascontiguousarray(ofs, np.int32)]
        w, o = keep[-2].ctypes.data, keep[-1].ctypes.data
    n_pts = 0 if pts is None else len(pts)
    n_traj = 0 if ofs is None else len(ofs) - 1
    return keep, (p, n_pts, w, o, n_traj, ctypes.c_float(VOXEL / 2), ctypes.c_float(2 * VOXEL))


def latency(ctx, args, reps):
    lib, h = ctx.lib, ctx.h
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        assert lib.dsm_field_query_enqueue(h, *args) == 0
        assert lib.dsm_field_query_wait(h, None, None) == 0
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def kernels(ctx, args, launches, n_samples, n_points):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib, h = ctx.lib, ctx.h
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            assert lib.dsm_field_query_enqueue(h, *args) == 0
            assert lib.dsm_field_query_wait(h, None, None) == 0
        torch.cuda.synchronize()
    out = {}
    for name, key, nbytes in (("k_field_query", "k_field_query", 72 * n_points), ("k_field_clearance", "k_field_clearance", 32 * n_samples)):
        rows = [k for k in prof.key_averages() if key in k.key]
        count = sum(k.count for k in rows)
        if count == 0:
            continue
        us = sum(k.device_time_total for k in rows) / count
        out[name] = {"launches": count, "us": us, "model_bytes": nbytes, "share_of_3.35TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}
    for name, key in (("h2d_copy", "Memcpy HtoD"), ("d2h_copy", "Memcpy DtoH")):
        rows = [k for k in prof.key_averages() if key in k.key]
        out[name] = {"us_per_query": sum(k.device_time_total for k in rows) / max(launches, 1)}
    return out


def host_numpy(host, pts, wp, ofs, reps):
    import pyoracle_field_query as fq
    dist, origin, _ = host
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        if pts is not None:
            fq.sample(dist, origin, VOXEL, pts)
        if wp is not None:
            fq.clearance(dist, origin, VOXEL, wp, ofs, VOXEL / 2, 2 * VOXEL)
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pyoracle_field_query as fq
    name, power = card()
    res = {"card": name, "power_limit": power, "grid": GRID, "voxel": VOXEL, "store_surfels": STORE, "queries": []}
    ctx, host = field_context()
    for label, pts, wp, ofs, n in cases(host[1]):
        keep, args = raw_args(pts, wp, ofs)
        n_samples = 0 if wp is None else len(fq.trajectory_samples(wp, ofs, VOXEL / 2)[0])
        for _ in range(5):   # warm-up
            assert ctx.lib.dsm_field_query_enqueue(ctx.h, *args) == 0 and ctx.lib.dsm_field_query_wait(ctx.h, None, None) == 0
        r = {"case": label, "n": n, "samples": n_samples, "latency_ms": latency(ctx, args, a.reps),
             "kernels": kernels(ctx, args, a.launches, n_samples, 0 if pts is None else len(pts)),
             "host_numpy_ms": host_numpy(host, pts, wp, ofs, a.host_reps)}
        del keep
        res["queries"].append(r)
        print(json.dumps(r), flush=True)
    ctx.close()
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, GRID, VOXEL)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_field_query.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
