"""Measure the viewpoint jobs (dsm_viewpoint_*, DESIGN.md §8.15) against scoring the same candidates as gain views.

Known fields of tools/measure_field_known.py's scene (eight 1226x370 frames captured into 256 slots) at 0.2 m, for every
--grids grid: the state grid is taken once and loaded (dsm_debug_field_load_state) into one context, a frontier job and
a reach job (host copy) from the scene's centre run on it, and a viewpoint job over the first --clusters clusters with
16 rotations (eight yaws level, eight pitched 15 degrees down), the 1226x370 camera at 25 voxels of range, offsets at
2 to 10 voxels with stride 2 and |dz| <= 2, top_k 4, with and without reach, at --samples samples per cluster.  For
each: the latency, host clock from dsm_viewpoint_enqueue to the end of dsm_viewpoint_wait on an idle stream (median,
min-max of --reps), and kernel times from torch.profiler in a run of their own.  Against that, the same reached
candidates and rotations scored as gain views naming the cluster, in as few gain requests as the gain work bound
allows, timed the same way, with the viewpoints each cluster whose members are all samples would get from those gains
checked equal to the job's; and the numpy model (oracle/pyoracle_viewpoint) on one cluster.  The card's name and power limit
are read in the same run.  Fails without a GPU.
Usage: python tools/measure_viewpoint.py [--grids 320x320x40 512x512x64] [--out DIR]"""
import argparse
import json
import math
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
from measure_drive import card, kernel_us, spread  # noqa: E402
from measure_field_known import MAX_RANGE, MAX_VIEWS, VOXEL, scene  # noqa: E402
import pyoracle_gain as G  # noqa: E402
import pyoracle_viewpoint as V  # noqa: E402

KERNELS = ["k_vp_clusters", "k_vp_candidates", "k_vp_score", "k_vp_select", "k_gain_init", "k_gain_views"]
CAM = synth.KITTI
RANGE_VOXELS = 25


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


def rotations():
    out = []
    for tilt in (0.0, np.deg2rad(15.0)):
        for k in range(8):
            a = 0.25 * math.pi * k
            f = np.array([math.cos(a) * math.cos(tilt), math.sin(a) * math.cos(tilt), -math.sin(tilt)])
            r = np.array([math.sin(a), -math.cos(a), 0.0])
            out.append(np.stack([r, np.cross(f, r), f], 1).reshape(9))
    return np.array(out)


def as_gain_views(ctx, state, origin, table, cl, rot, prm, cost, gc):
    """The reached candidates of each cluster as gain views, one per rotation, in requests within the gain work bound:
    (function running them all, function turning their gains into the (cluster, ranked slots) the job would return)."""
    nz, ny, nx = state.shape
    off = V.offsets(prm)
    trav = state == G.FREE
    views, meta = [], []
    for i, c in enumerate(cl):
        g = V.centre_voxel(table[c]["centroid"], origin, VOXEL)
        for j, o in enumerate(off):
            x, y, z = g + o
            if not (0 <= x < nx and 0 <= y < ny and 0 <= z < nz) or not trav[z, y, x]:
                continue
            if prm.with_reach and cost[z, y, x] == V.INF:
                continue
            t = G.centres([(x, y, z)], origin, VOXEL)[0]
            for r, R in enumerate(rot):
                views.append(np.concatenate([R.reshape(3, 3), t[:, None]], 1).reshape(12))
                meta.append((i, j, r, int((z * ny + y) * nx + x), int(cost[z, y, x]) if prm.with_reach else V.INF))
    views = np.array(views).reshape(-1, 12)
    named = np.array([cl[m[0]] for m in meta], np.int32)
    m = 2 * math.ceil(float(np.float32(gc.max_range)) / float(np.float32(VOXEL))) + 3
    per = max(1, min(G.MAX_WORK // m ** 3, 1 << 14))

    def run():
        out = []
        for a in range(0, len(views), per):
            ctx.gain_enqueue(gc, views[a:a + per], named[a:a + per])
            out.append(ctx.gain_wait()[1]["n_cluster"])
        return np.concatenate(out) if out else np.zeros(0, np.int32)

    def rank(n_cluster):
        best = {}
        for (i, j, r, vox, c), n in zip(meta, n_cluster):
            if (i, j) not in best or n > best[(i, j)][0]:
                best[(i, j)] = (int(n), c, j, r, vox)
        slots = [[] for _ in cl]
        for (i, j), (n, c, jj, r, vox) in best.items():
            if n >= max(1, prm.min_seen):
                slots[i].append((-n, c, jj, r, vox))
        return [sorted(s)[:prm.top_k] for s in slots]
    return run, rank, len(views)


def measure(state, origin, centre, grid, a):
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(4096, 1 << 20)
    ctx.reach_enable(16, 1 << 12, 4096)
    ctx.gain_enable(1 << 14)
    ctx.viewpoint_enable(4096, 1 << 22)
    ctx.debug_field_load_state(state, origin)
    dist = ctx.field_wait()[0]
    ctx.frontier_enqueue(1)
    fc, fv, _ = ctx.frontier_wait()
    ctx.reach_enqueue(centre, 0.0, 2, None, False, True)
    cost = ctx.reach_wait()[3]
    cl = np.arange(min(a.clusters, len(fc)), dtype=np.int32)
    rot = rotations()
    gc = G.Camera(CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.width, CAM.height, float(np.float32(RANGE_VOXELS * VOXEL)), 1)
    r = {"grid": grid, "clusters_in_table": len(fc), "clusters": len(cl), "rotations": len(rot), "jobs": []}
    for with_reach in (0, 1):
        for samples in a.samples:
            prm = V.Params(2, 10, 2, 2, samples, 1, 4, with_reach, 0.0)

            def job():
                ctx.viewpoint_enqueue(gc, rot, cl, prm)
                return ctx.viewpoint_wait()
            info, recs, slots = job()
            e = {"with_reach": with_reach, "max_samples": samples, "offsets": int(info["n_offsets"]),
                 "reached_candidates": int(recs["n_reached"].sum()), "samples": int(recs["n_samples"].sum()),
                 "viewpoints": int(recs["n_viewpoints"].sum()), "latency_ms": timed(job, a.reps, ctx)}
            per = kernel_us(lambda: [job() for _ in range(a.launches)], KERNELS)
            e["kernels_us"] = {k: sum(v) / a.launches for k, v in per.items() if v}
            if samples >= 4096:
                run, rank, n_views = as_gain_views(ctx, state, origin, fc, cl, rot, prm, cost, gc)
                got = [[(-int(s["n_seen"]), int(s["cost"]), int(s["offset"]), int(s["rotation"]), int(s["voxel"]))
                        for s in slots[i] if s["voxel"] >= 0] for i in range(len(cl))]
                full = [i for i in range(len(cl)) if recs[i]["n_samples"] == fc[cl[i]]["n_voxels"]]
                want = rank(run())
                assert [want[i] for i in full] == [got[i] for i in full], "gain views and the viewpoint job differ"
                e["as_gain_views"] = {"views": n_views, "clusters_checked": len(full), "latency_ms": timed(run, a.reps, ctx)}
                per = kernel_us(lambda: [run() for _ in range(a.launches)], KERNELS)
                e["as_gain_views"]["kernels_us"] = {k: sum(v) / a.launches for k, v in per.items() if v}
                t0 = time.perf_counter()
                want = V.viewpoints(state, dist, origin, VOXEL, gc, rot, cl[:1], prm, (fc, fv), cost if with_reach else None)
                e["host_model_ms_one_cluster"] = (time.perf_counter() - t0) * 1e3
                ctx.viewpoint_enqueue(gc, rot, cl[:1], prm)
                one = ctx.viewpoint_wait()
                assert all(x.tobytes() == np.asarray(y).tobytes() for x, y in zip(one, want)), "device and model differ"
            r["jobs"].append(e)
            print(json.dumps(e), flush=True)
    ctx.close()
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["320x320x40", "512x512x64"])
    ap.add_argument("--clusters", type=int, default=111)
    ap.add_argument("--samples", type=int, nargs="+", default=[64, 4096])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "camera": [CAM.width, CAM.height], "known": []}
    for gs in a.grids:
        grid = tuple(int(x) for x in gs.split("x"))
        ctx, poses, views, c = scene()
        ctx.field_enable(VOXEL, *grid)
        ctx.views_enable(MAX_VIEWS, MAX_RANGE)
        for j in range(MAX_VIEWS):
            ctx.views_capture(j % 8, j)
        ctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses)
        origin = ctx.field_wait()[1]
        state = ctx.field_state()[0].copy()
        ctx.close()
        res["known"].append(measure(state, origin, c, grid, a))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_viewpoint.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
