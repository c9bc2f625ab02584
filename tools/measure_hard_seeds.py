"""Share of "hard" Huber-Newton seeds per update pass on the bench.py frames.

k_gather runs the Newton of every updated seed as long as all of its member depths are inside the Huber range; a seed
that meets an out-of-range entry is queued for k_newton_hard, which is what remains of the Newton phase after k_gather.
This script stops the schedule after each pass's assign (dsm_debug_stop_after), reads the labels and stable flags, and
replays each updated seed's mean and in-range Newton passes on the host in float32, entry by entry as the kernel does,
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

F32 = np.float32
DEPTH_MIN = np.array(0x3dcccccc, np.uint32).view(np.float32)  # (double)depth > 0.1  <=>  depth > this float
DELTA_HI = np.array(0x3c23d70b, np.uint32).view(np.float32)   # |(double)delta| < 0.01  <=>  |delta| < this float


def huber_hi(h):
    f = F32(h)
    return f if float(f) >= h else np.nextafter(f, F32(np.inf))


def is_hard(z, hh):
    """True if the Newton of a seed with member depths z (raster order, float32) meets an out-of-range entry."""
    nd = len(z)
    md = F32(np.cumsum(z, dtype=F32)[-1] / F32(nd))  # sequential float sum, as the kernel's mean pass
    zmn, zmx = z.min(), z.max()
    for _ in range(5):
        if not ((md - zmn) < hh and (md - zmx) > -hh):
            return True
        sa = np.cumsum(F32(2) * (md - z), dtype=F32)[-1]  # fmaf(2, md - z, sa): 2 r is exact
        delta = F32(-float(sa) / (float(2 * nd) + 10.0))
        md = F32(md + delta)
        if -DELTA_HI < delta < DELTA_HI:
            return False
    return False


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
    W, H = cam.width, cam.height
    spw, sph = W // 8, H // 8
    hh = huber_hi(capi.CONSTANTS_DRIVE[0])  # a fresh context holds the drive constants
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=16)
    ctx.batch_upload([0] * B, gray, depth, poses, np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    passes = []
    for it in range(3):
        ctx.debug_stop_after(2 + 3 * it)  # seed init, then (assign, gather, Newton) per pass: stop after this pass's assign
        ctx.batch_run()
        ctx.sync()
        upd = hard = entries = hard_entries = 0
        for b in range(B):
            lab, stable = ctx.labels(b), ctx.seeds(b)["stable"]
            for s in np.nonzero(stable == 0)[0]:
                sy, sx = divmod(int(s), spw)
                x0, y0 = sx * 8 - 4, sy * 8 - 4
                xb, yb, xe, ye = max(x0, 0), max(y0, 0), min(x0 + 16, W - 1), min(y0 + 16, H - 1)
                z = depth[b, yb:ye, xb:xe]
                z = z[(lab[yb:ye, xb:xe] == s) & (z > DEPTH_MIN)]
                upd += 1
                entries += len(z)
                if len(z) and is_hard(z, hh):
                    hard += 1
                    hard_entries += len(z)
        passes.append({"pass": it + 1, "updated_seeds": upd, "hard_seeds": hard, "hard_share": hard / max(upd, 1),
                       "entries": entries, "hard_entries": hard_entries, "hard_entry_share": hard_entries / max(entries, 1)})
        print(json.dumps(passes[-1]), flush=True)
    ctx.debug_stop_after(0)
    ctx.close()
    res = {"frames": B, "seeds_per_frame": spw * sph, "passes": passes}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "hard_seeds.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
