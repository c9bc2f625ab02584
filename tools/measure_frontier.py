"""Measure the exploration frontiers (dsm_frontier_*, DESIGN.md §8.10) against the host path a planner uses without them.

1. Known fields of tools/measure_field_known.py's scene (eight 1226x370 frames captured into 256 slots) at 0.2 m, for
   every --grids grid and --views count: the job's latency, host clock from dsm_frontier_enqueue to the end of
   dsm_frontier_wait on an idle stream (median, min-max of --reps), and its kernels from torch.profiler.  Against that,
   the host path: the state grid's D2H copy (a host-copy known request minus a resident one, both waited for), then
   oracle/pyoracle_frontier (numpy marking, scipy.ndimage.label and the statistics) on the host copy.
2. The same on loaded adversarial 320x320x40 grids (dsm_debug_field_load_state): 50 % free / 50 % unknown at random,
   and the serpentine of tests/test_frontier_model.py.
3. The node drive of tools/measure_node.py (tools/measure_frontier.cpp), modes alternating on fresh nodes, --rounds
   rounds, a 320x320x40 known field (256 slots, rays cut at 40 m) read after every fuse: k known space alone; f with
   frontiers(1) after every fuse as well.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_frontier.py [--frames 320] [--rounds 3] [--out DIR]"""
import argparse
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import build_harness, card, images, kernel_us, messages, run_harness, spread, write_drive  # noqa: E402
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
import pyoracle_frontier  # noqa: E402
from test_frontier_model import serpentine  # noqa: E402

CAPS = (4096, 1 << 20)
KERNELS = ["k_frontier_mark", "k_frontier_tile", "k_frontier_seam", "k_frontier_flatten", "k_frontier_sel", "k_frontier_number",
           "k_frontier_count", "k_frontier_keep", "k_frontier_slot", "k_frontier_reduce", "k_frontier_table", "k_frontier_keys",
           "DeviceScan", "DeviceRadixSort"]


def timed(fn, reps, ctx):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def job(ctx):
    ctx.frontier_enqueue(1)
    return ctx.frontier_wait()


def kernels(ctx, launches):
    per = kernel_us(lambda: [job(ctx) for _ in range(launches)], KERNELS)
    return {k: sum(v) / launches for k, v in per.items() if v}


def host_path(state, origin, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        pyoracle_frontier.frontiers(state, origin, VOXEL, 1, *CAPS)
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def measure(ctx, reps, launches, request, what, copies=True):
    """request(host_copy) makes the latest field; the record of the job on it against the host path."""
    request(True)
    _, origin, _ = ctx.field_wait()
    state, _ = ctx.field_state()
    got = job(ctx)
    want = pyoracle_frontier.frontiers(state, origin, VOXEL, 1, *CAPS)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(got, want)), f"{what}: device and model differ"
    r = {"what": what, "counts": {n: int(got[2][n]) for n in got[2].dtype.names}, "latency_ms": timed(lambda: job(ctx), reps, ctx)}
    r["kernels_us"] = kernels(ctx, launches)
    r["kernel_sum_us"] = sum(r["kernels_us"].values())
    r["host_numpy_ms"] = host_path(state, origin, max(3, reps // 5))
    if copies:   # the state grid's D2H: a host-copy known request against a resident one, each waited for

        def field(host):
            request(host)
            ctx.field_wait()
        r["field_request_ms"] = {"host_copy": timed(lambda: field(True), reps, ctx), "resident": timed(lambda: field(False), reps, ctx)}
    print(json.dumps(r), flush=True)
    return r


def node_drive(n_frames, rounds, grid):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_harness(tmp, "measure_frontier")
        ff, fs = write_drive(tmp, images(), messages(n_frames))
        times = {m: [] for m in "kf"}
        last = {}
        for _ in range(rounds):
            for m in "kf":
                last[m] = run_harness(exe, ff, fs, [m, VOXEL, *grid, MAX_VIEWS, MAX_RANGE])
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "clusters_per_frame": last["f"]["clusters"] / n_frames,
            "listed_per_frame": last["f"]["listed"] / n_frames, "ms_per_frame": {m: spread(times[m]) for m in "kf"}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--views", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--node-grid", default="320x320x40")
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "caps": CAPS, "known": [], "loaded": []}
    for g in a.grids:
        grid = tuple(int(x) for x in g.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        ctx.frontier_enable(*CAPS)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)
        for n in a.views:
            def request(host, n=n):
                ctx.field_enqueue_known(c, 5, list(range(n)), poses[:n], host_copy=host)
            res["known"].append({"grid": grid, "views": n, **measure(ctx, a.reps, a.launches, request, f"{g} {n} views")})
        ctx.close()
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    grid = (320, 320, 40)
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(*CAPS)
    rng = np.random.default_rng(1)
    for what, st in [("random 50 % free", rng.choice([0, 2], size=grid[::-1]).astype(np.uint8)), ("serpentine", serpentine(*grid))]:
        def request(host, st=st):
            ctx.debug_field_load_state(st, (-160, -160, -5))
        res["loaded"].append(measure(ctx, a.reps, a.launches, request, what, copies=False))
    ctx.close()
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, tuple(int(x) for x in a.node_grid.split("x")))
        print(json.dumps(res["node_drive"]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_frontier.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
