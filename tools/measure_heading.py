"""Measure the heading jobs (dsm_heading_*, DESIGN.md §8.19) against scoring the same (sample, rotation) poses as gain
views.

The known field of tools/measure_field_known.py's scene (eight 1226x370 frames captured into 256 slots) at 0.2 m on a
--grid grid is taken once and loaded (dsm_debug_field_load_state) into one context.  For 1, 16 and 64 trajectories of
16 to 64 control points (seeded noisy lines of 6 to 20 m through the scene's centre), K = 4 samples per segment, 8 and
16 yaws and 25 and 50 voxels of range with the 1226x370 camera: the latency, host clock from dsm_heading_enqueue to the
end of dsm_heading_wait on an idle stream (median, min-max of --reps), and k_heading_views and k_heading_plan from
torch.profiler in a run of their own.  Against that, the same S x R poses as gain views, timed the same way and their
n_unknown and n_frontier checked equal to the heading job's counts.  A request beyond either job's work bound of 2^31
voxel visits is split into as few calls as the bound allows, and the times add up.  The card's name and power limit
are read in the same run.  Fails without a GPU.
Usage: python tools/measure_heading.py [--grid 320x320x40] [--reps N] [--out DIR]"""
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
import pyoracle_heading as H  # noqa: E402

KERNELS = ["k_heading_views", "k_heading_plan", "k_gain_init", "k_gain_views"]
CAM = synth.KITTI
K = 4


def yaws(n):
    out = []
    for k in range(n):
        a = 2 * math.pi * k / n
        f, r = np.array([math.cos(a), math.sin(a), 0.0]), np.array([math.sin(a), -math.cos(a), 0.0])
        out.append(np.stack([r, np.cross(f, r), f], 1).reshape(9))
    return np.array(out)


def trajectories(rng, n, centre):
    pts, ofs = [], [0]
    for _ in range(n):
        N = int(rng.integers(16, 65))
        d = rng.standard_normal(3) * [1.0, 1.0, 0.1]
        d *= rng.uniform(3.0, 10.0) / np.linalg.norm(d)
        pts.append(centre + np.linspace(-1, 1, N)[:, None] * d + rng.standard_normal((N, 3)) * 0.1)
        ofs.append(ofs[-1] + N)
    return np.concatenate(pts), np.array(ofs, np.int32)


def chunks(sizes, per_call):
    """Consecutive index ranges of `sizes` whose sums stay within per_call."""
    out, a, tot = [], 0, 0
    for i, s in enumerate(sizes):
        if tot + s > per_call and i > a:
            out.append((a, i))
            a, tot = i, 0
        tot += s
    out.append((a, len(sizes)))
    return out


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


def measure(ctx, n_traj, n_rot, range_voxels, rng, centre, reps):
    pts, ofs = trajectories(rng, n_traj, centre)
    rot = yaws(n_rot)
    gc = G.Camera(CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.width, CAM.height, float(np.float32(range_voxels * VOXEL)), 1)
    m3 = (2 * range_voxels + 3) ** 3
    lens = np.diff(ofs)
    S = K * (lens - 3) + 1
    req = H.requests([(0, -1, 1)] * n_traj)
    head_calls = chunks(S, H.MAX_WORK // m3)
    out = {}

    def heading():
        for a, b in head_calls:
            ctx.heading_enqueue(pts[ofs[a]:ofs[b]], ofs[a:b + 1] - ofs[a], gc, rot, K, req[a:b], 1, 1)
            out.setdefault("heading", []).append(ctx.heading_wait())

    pos = H.sample_positions(pts, ofs, K)
    poses = np.array([np.concatenate([R.reshape(3, 3), p[:, None]], 1).reshape(12) for p in pos for R in rot])
    gain_calls = chunks(np.ones(len(poses), np.int64), min(G.MAX_WORK // m3, G.MAX_VIEWS))

    def gain():
        for a, b in gain_calls:
            ctx.gain_enqueue(gc, poses[a:b])
            out.setdefault("gain", []).append(ctx.gain_wait()[1])

    heading()
    gain()
    counts = np.concatenate([h[3].reshape(-1) for h in out["heading"]])
    g = np.concatenate(out["gain"])
    assert (g["n_unknown"] == counts["n_unknown"]).all() and (g["n_frontier"] == counts["n_frontier"]).all(), "counts"
    row = dict(trajectories=n_traj, points=int(ofs[-1]), samples=int(len(pos)), rotations=n_rot, range_voxels=range_voxels,
               heading_calls=len(head_calls), gain_calls=len(gain_calls), seen_unknown=int(counts["n_unknown"].sum()))
    row["heading_ms"] = timed(heading, reps, ctx)
    row["gain_ms"] = timed(gain, reps, ctx)
    ku = kernel_us(heading, KERNELS[:2])
    kg = kernel_us(gain, KERNELS[2:])
    row["kernels_us"] = {k: float(sum(v)) for k, v in {**ku, **kg}.items()}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grid", default="320x320x40")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    grid = tuple(int(x) for x in a.grid.split("x"))
    sctx, poses, views, c = scene()
    sctx.field_enable(VOXEL, *grid)
    sctx.views_enable(MAX_VIEWS, MAX_RANGE)
    for j in range(MAX_VIEWS):
        sctx.views_capture(j % 8, j)
    sctx.field_enqueue_known(c, 5, list(range(MAX_VIEWS)), poses)
    origin = sctx.field_wait()[1]
    state = sctx.field_state()[0].copy()
    sctx.close()
    ctx = capi.Context(synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0), max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(VOXEL, *grid)
    ctx.views_enable(1, 1.0)
    ctx.heading_enable(64, 1 << 16)
    ctx.gain_enable(G.MAX_VIEWS)
    ctx.debug_field_load_state(state, origin)
    ctx.field_wait()
    res = {"card": name, "power_limit": power, "voxel": VOXEL, "grid": list(grid), "camera": [CAM.width, CAM.height], "K": K,
           "runs": []}
    rng = np.random.default_rng(1)
    for n_traj in (1, 16, 64):
        for n_rot in (8, 16):
            for rv in (25, 50):
                res["runs"].append(measure(ctx, n_traj, n_rot, rv, rng, np.asarray(c, np.float64), a.reps))
    ctx.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_heading.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
