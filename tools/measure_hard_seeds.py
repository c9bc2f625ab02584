"""Share of "hard" Huber-Newton seeds per update pass on the bench.py frames.

k_gather runs the Newton of every updated seed as long as all of its member depths are inside the Huber range; a seed
that meets an out-of-range entry is queued for k_newton_hard, which is what remains of the Newton phase after k_gather.
This script stops the schedule after each pass's assign (dsm_debug_stop_after), reads the labels and stable flags, and
replays each updated seed's update on the host (oracle/pyoracle_newton.py: float32, entry by entry as the reference)
to count the seeds k_gather queues.  Needs a GPU.
Usage: python tools/measure_hard_seeds.py [--frames N] [--out DIR]   (writes DIR/hard_seeds.json when --out is given)
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import make_batch  # noqa: E402
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyoracle_newton as pn  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cam = synth.KITTI
    B = args.frames
    _, cur = make_batch(cam, 32, 0)  # the bench.py frames; the first B are measured
    cur = cur[:B]
    gray, depth = np.stack([f[0] for f in cur]), np.stack([f[1] for f in cur])
    poses = np.stack([f[2] for f in cur]).astype(np.float32)
    huber = capi.CONSTANTS_DRIVE[0]  # a fresh context holds the drive constants
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=16)
    ctx.batch_upload([0] * B, gray, depth, poses, np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    passes = []
    for it in range(3):
        ctx.debug_stop_after(2 + 3 * it)  # seed init, then (assign, gather, Newton) per pass: stop after this pass's assign
        ctx.batch_run()
        ctx.sync()
        upd = hard = entries = hard_entries = 0
        for b in range(B):
            rep = pn.replay(ctx.labels(b), ctx.seeds(b), depth[b], huber)
            u, q = rep["branch"] != pn.SKIPPED, rep["branch"] == pn.QUEUED
            upd += int(u.sum())
            hard += int(q.sum())
            entries += int(rep["nd"][u].sum())
            hard_entries += int(rep["nd"][q].sum())
        passes.append({"pass": it + 1, "updated_seeds": upd, "hard_seeds": hard, "hard_share": hard / max(upd, 1),
                       "entries": entries, "hard_entries": hard_entries, "hard_entry_share": hard_entries / max(entries, 1)})
        print(json.dumps(passes[-1]), flush=True)
    ctx.debug_stop_after(0)
    ctx.close()
    res = {"frames": B, "seeds_per_frame": ctx.S, "passes": passes}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "hard_seeds.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
