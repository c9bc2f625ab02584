"""Measure the reach jobs (dsm_reach_*, DESIGN.md §8.11) against the host path a planner uses without them.

1. Known fields of tools/measure_field_known.py's scene (eight 1226x370 frames captured into 256 slots) at 0.2 m, for
   every --grids grid: the state grid is taken once and loaded (dsm_debug_field_load_state) into contexts enabled with
   each --max-rounds, so every job runs on the same field.  A job starts at the scene's centre (radius one voxel,
   approach 2) toward the frontier clusters of frontiers(1) and --goals random goals.  Per max_rounds: the latency, host
   clock from dsm_reach_enqueue to the end of dsm_reach_wait on an idle stream (median, min-max of --reps), rounds and
   converged; the empty-round tail is the latency difference between two caps that both converge, per empty round.
   Kernels from torch.profiler at the smallest converging cap.  Against that, the host path: both grids' D2H copy (a
   host-copy known request minus a resident one, both waited for), scipy's Dijkstra (oracle/pyoracle_reach) and the
   target matching (the windows of every goal and cluster member on the host).
2. The same on loaded adversarial 320x320x40 grids: 50 % free / 50 % occupied at random, and the serpentine of
   tests/test_frontier_model.py (one corridor of about a million voxels: it does not converge within 65536 rounds).
3. The node drive of tools/measure_node.py (tools/measure_reach.cpp), modes alternating on fresh nodes, --rounds rounds,
   a 320x320x40 known field read after every fuse: f with frontiers(1) after every fuse; r with reach(with_frontiers)
   from the camera's voxel as well, at --node-max-rounds.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_reach.py [--frames 320] [--rounds 3] [--out DIR]"""
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
import pyoracle_reach  # noqa: E402
from test_frontier_model import serpentine  # noqa: E402

FRONTIER_CAPS = (4096, 1 << 20)
CAPS = (4096, 1 << 18)
KERNELS = ["k_reach_start", "k_reach_init", "k_reach_round", "k_reach_settle", "k_reach_reached", "k_reach_targets", "k_reach_records",
           "k_reach_paths", "DeviceScan"]


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


def loader(grid, max_rounds):
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(*FRONTIER_CAPS)
    ctx.reach_enable(*CAPS, max_rounds)
    return ctx


def host_path(state, dist, origin, start, goals, fr):
    """scipy's Dijkstra on the host copy, then the target matching (every goal's and member's window)."""
    trav = pyoracle_reach.traversable(state, dist, VOXEL)
    nz, ny, nx = state.shape
    t0 = time.perf_counter()
    s = pyoracle_reach.voxel_of(start, origin, VOXEL, (nx, ny, nz))
    u, _, _ = pyoracle_reach.snap(trav, s, 2)
    cost = pyoracle_reach.dijkstra(trav, u)
    t1 = time.perf_counter()
    for g in goals:
        pyoracle_reach.best_in_window(trav, cost, pyoracle_reach.voxel_of(g, origin, VOXEL, (nx, ny, nz)), 2)
    for gi in fr[1].tolist():
        pyoracle_reach.best_in_window(trav, cost, (gi % nx, gi // nx % ny, gi // (nx * ny)), 2)
    t2 = time.perf_counter()
    return {"dijkstra_ms": (t1 - t0) * 1e3, "matching_ms": (t2 - t1) * 1e3, "members": len(fr[1])}, cost


def measure(state, origin, start, goals, caps_rounds, reps, launches, what, host=True):
    grid = state.shape[::-1]
    r = {"what": what, "grid": grid, "by_max_rounds": []}
    ref = None
    for mr in caps_rounds:
        ctx = loader(grid, mr)
        ctx.debug_field_load_state(state, origin)
        dist = ctx.field_wait()[0]
        ctx.frontier_enqueue(1)
        fr = ctx.frontier_wait()

        def job():
            ctx.reach_enqueue(start, VOXEL, 2, goals, True, False)
            return ctx.reach_wait()
        info, targets, path, _ = job()
        e = {"max_rounds": mr, "rounds": int(info["rounds"]), "converged": int(info["converged"]),
             "n_traversable": int(info["n_traversable"]), "n_reached": int(info["n_reached"]), "n_targets": int(info["n_targets"]),
             "reached_targets": int((targets["status"] == 0).sum()), "n_path_voxels": int(info["n_path_voxels"]),
             "latency_ms": timed(job, reps, ctx)}
        if info["converged"] and ref is None:
            ref = mr
            per = kernel_us(lambda: [job() for _ in range(launches)], KERNELS)
            e["kernels_us"] = {k: sum(v) / launches for k, v in per.items() if v}
            e["round_launches"] = len(per["k_reach_round"]) // launches
            if host:
                ctx.reach_enqueue(start, VOXEL, 2, goals, True, True)
                cost = ctx.reach_wait()[3]
                h, want = host_path(state, dist, origin, start, goals, fr)
                assert cost.tobytes() == want.tobytes(), f"{what}: device and Dijkstra differ"
                r["host"] = h
        r["by_max_rounds"].append(e)
        print(json.dumps(e), flush=True)
        ctx.close()
    conv = [e for e in r["by_max_rounds"] if e["converged"]]
    if len(conv) >= 2:
        a, b = conv[0], conv[-1]
        r["empty_round_us"] = (b["latency_ms"]["median"] - a["latency_ms"]["median"]) * 1e3 / (b["max_rounds"] - a["max_rounds"])
    print(json.dumps({k: v for k, v in r.items() if k != "by_max_rounds"}), flush=True)
    return r


def copies(grid, request, ctx, reps):
    """Both grids' D2H copy: a host-copy known request against a resident one, each waited for."""
    def field(host):
        request(host)
        ctx.field_wait()
    return {"host_copy": timed(lambda: field(True), reps, ctx), "resident": timed(lambda: field(False), reps, ctx)}


def node_drive(n_frames, rounds, grid, max_rounds):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_harness(tmp, "measure_reach")
        ff, fs = write_drive(tmp, images(), messages(n_frames))
        times = {m: [] for m in "fr"}
        last = {}
        for _ in range(rounds):
            for m in "fr":
                last[m] = run_harness(exe, ff, fs, [m, VOXEL, *grid, MAX_VIEWS, MAX_RANGE, max_rounds])
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "grid": grid, "max_rounds": max_rounds,
            "reached_targets_per_frame": last["r"]["reached"] / n_frames, "converged_frames": last["r"]["converged"],
            "most_rounds": last["r"]["most_rounds"], "ms_per_frame": {m: spread(times[m]) for m in "fr"}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--max-rounds", type=int, nargs="+", default=[16, 64, 256, 1024, 4096])
    ap.add_argument("--goals", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--node-grid", default="320x320x40")
    ap.add_argument("--node-max-rounds", type=int, default=64)
    ap.add_argument("--skip-node", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "caps": CAPS, "known": [], "loaded": []}
    rng = np.random.default_rng(3)
    for g in a.grids:
        grid = tuple(int(x) for x in g.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)

        def request(host):
            ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses, host_copy=host)
        request(True)
        origin = ctx.field_wait()[1]
        state = ctx.field_state()[0].copy()
        cp = copies(grid, request, ctx, a.reps)
        ctx.close()
        goals = c + rng.uniform(-1, 1, size=(a.goals, 3)) * np.array(grid) * VOXEL * 0.4
        r = measure(state, origin, c, goals, a.max_rounds, a.reps, a.launches, f"{g} scene")
        r["field_request_ms"] = cp
        res["known"].append(r)
    grid = (320, 320, 40)
    o = (-160, -160, -5)
    start = ((o[0] + 0.5) * VOXEL, (o[1] + 0.5) * VOXEL, (o[2] + 0.5) * VOXEL)
    goals = [((o[0] + grid[0] - 0.5) * VOXEL, (o[1] + grid[1] - 0.5) * VOXEL, (o[2] + k + 0.5) * VOXEL) for k in range(0, 40, 8)]
    for what, st, host in [("random 50 % free", rng.choice([1, 2], size=grid[::-1]).astype(np.uint8), True),
                           ("serpentine", serpentine(*grid), False)]:
        st[0, 0, 0] = 2
        res["loaded"].append(measure(st, o, start, goals, a.max_rounds, a.reps, a.launches, what, host))
    if not a.skip_node:
        res["node_drive"] = node_drive(a.frames, a.rounds, tuple(int(x) for x in a.node_grid.split("x")), a.node_max_rounds)
        print(json.dumps(res["node_drive"]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_reach.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
