"""Views in the checkpoint (DESIGN.md §8.18) on one GPU, with 1226x370 frames (7 038 rays per view) and 256 slots:
enqueue to durable file of a full dsm_checkpoint_enqueue with 0 and with 256 filled slots, the size and enqueue to
durable record of an incremental checkpoint that adds one view, and dsm_map_load of the 256-view file.  Prints one JSON
object with the card's name and power limit, read in the same run.
Usage: python tools/measure_checkpoint_views.py [--reps N] [--out DIR]"""
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
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from measure_drive import card, spread  # noqa: E402

CAM = synth.KITTI
SLOTS = 256


def context():
    """A resident 1226x370 context with one fused frame, a field, 256 view slots and view checkpoints."""
    ctx = capi.Context(CAM, max_batch=2, max_local_surfels=1 << 20)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.inactive_reserve(1 << 20)
    ctx.field_enable(0.2, 64, 64, 32)
    ctx.views_enable(SLOTS, 30.0)
    ctx.checkpoint_enable()
    ctx.checkpoint_views_enable()
    gray, depth = synth.make_frame(CAM, 7, synth.pose_stream(0))
    ctx.fuse_frame_resident(0, gray, depth, synth.pose_stream(0))
    ctx.sync()
    return ctx


def timed(fn, reps):
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t) * 1e3)
    return spread(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    d = tempfile.mkdtemp(prefix="dsm_views_")
    ctx = context()
    res = {"card": name, "power_limit": power, "rays_per_view": capi.load_library().dsm_num_seeds(ctx.h), "slots": SLOTS}

    def full(path):
        ctx.checkpoint_enqueue(path)
        ctx.checkpoint_wait(True)

    p0 = os.path.join(d, "empty.dsm")
    res["full_0_views_ms"] = timed(lambda: full(p0), a.reps)
    res["full_0_views_bytes"] = os.path.getsize(p0)
    for s in range(SLOTS):
        ctx.views_capture(0, s)
    p256 = os.path.join(d, "full.dsm")
    full(p256)   # the first snapshot after the captures copies all 256 slots into the image
    res["full_256_views_first_ms"] = timed(lambda: full(p256), 1)
    res["full_256_views_ms"] = timed(lambda: full(p256), a.reps)
    res["full_256_views_bytes"] = os.path.getsize(p256)

    pj = os.path.join(d, "chain.dsm")
    ctx.checkpoint_enqueue_incremental(pj)
    ctx.checkpoint_wait(True)
    rec_ms, rec_bytes = [], []
    for k in range(a.reps):
        before = os.path.getsize(pj + ".journal")
        ctx.views_capture(0, k % SLOTS)
        t = time.perf_counter()
        ctx.checkpoint_enqueue_incremental(pj)
        ctx.checkpoint_wait(True)
        rec_ms.append((time.perf_counter() - t) * 1e3)
        rec_bytes.append(os.path.getsize(pj + ".journal") - before)
    res["record_one_view_ms"], res["record_one_view_bytes"] = spread(rec_ms), rec_bytes

    other = context()
    res["load_256_views_ms"] = timed(lambda: other.map_load(p256), a.reps)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "checkpoint_views.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
