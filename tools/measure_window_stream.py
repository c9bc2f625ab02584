"""Cost of the node's per-frame sequence (move_add_surfels + fuse_map) on the GPU-resident map, three ways.

A 1226x370 drive (synth.KITTI) with a keyframe every 4 frames, each frame referenced to the newest keyframe, and a
drift-free window of W keyframes along the chain (W = 3 and 10), with the inactive store reserved:
  per_call    dsm_fuse_frame_resident, with the synchronising dsm_inactive_retire / dsm_inactive_reactivate in front
              of every frame whose window changes (the recipe before dsm_fuse_stream_window)
  window_n1   dsm_fuse_stream_window, one frame per call
  window_nK   dsm_fuse_stream_window, K = 8 and 16 frames per call
The three run alternately, `--rounds` times each, on fresh contexts; ms per frame is the median over the rounds (host
clock from a synchronised start to the synchronise after the last frame).  A separate run under torch.profiler sums
the window step's own kernels (k_win_*).  Prints one JSON line per (window, mode) and one with the GPU's name and power limit.

  python tools/measure_window_stream.py [--frames 128] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402

CAM = synth.KITTI
N_IMG = 32  # distinct image pairs, cycled over the drive
KF_EVERY = 4


def window_lists(n_frames, window):
    """get_add_remove_poses along the drive (surfel_map.cpp:1597-1680): keyframe k is linked to k - 1 (its reference
    when it was created), the reference of frame f is the newest keyframe f // 4, the drift-free set is the BFS of depth
    `window` from it, i.e. keyframes root - window + 1 .. root.  A new keyframe joins local_surfels_indexs at once."""
    local, out = set(), []
    for f in range(n_frames):
        root = f // KF_EVERY
        local.add(root)
        free = list(range(root, max(-1, root - window), -1))
        add = [p for p in free if p not in local]
        rem = [p for p in sorted(local) if p not in free]
        local = (local - set(rem)) | set(add)
        out.append((root, rem, add))
    return out


def new_ctx(max_batch):
    ctx = capi.Context(CAM, max_batch=max_batch, max_local_surfels=2_000_000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.inactive_reserve(4_000_000)
    return ctx


def run(mode, chunk, lists, G, D, P, warm=16):
    """ms per frame of frames [warm, len(lists)) in one of the three ways; the first `warm` frames are not timed."""
    ctx = new_ctx(max_batch=32)

    def frames(f0, f1):
        if mode == "per_call":
            for f in range(f0, f1):
                ref, rem, add = lists[f]
                for kf in rem:
                    ctx.inactive_retire(kf)
                for kf in add:
                    ctx.inactive_reactivate(kf)
                ctx.fuse_frame_resident(ref, G[f % N_IMG], D[f % N_IMG], P[f])
            return
        for c0 in range(f0, f1, chunk):
            c1 = min(f1, c0 + chunk)
            i0 = c0 % N_IMG
            part = lists[c0:c1]
            ctx.fuse_stream_window([p[0] for p in part], G[i0:i0 + c1 - c0], D[i0:i0 + c1 - c0], P[c0:c1],
                                   [p[1] for p in part], [p[2] for p in part])

    frames(0, warm)
    ctx.pool_size()  # synchronises with the resident state
    t0 = time.perf_counter()
    frames(warm, len(lists))
    ctx.pool_size()  # waits for the last frame (and reports a rejected one)
    ms = (time.perf_counter() - t0) * 1e3 / (len(lists) - warm)
    n_pool, (n_store, n_seg) = ctx.pool_size(), ctx.inactive_size()
    ctx.close()
    return ms, n_pool, n_store, n_seg


def window_kernel_ms(lists, G, D, P, chunk=16):
    """Device time of the window step's kernels per frame that has one, from a run under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    ctx = new_ctx(max_batch=32)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c0 in range(0, len(lists), chunk):
            i0 = c0 % N_IMG
            part = lists[c0:c0 + chunk]
            ctx.fuse_stream_window([p[0] for p in part], G[i0:i0 + len(part)], D[i0:i0 + len(part)], P[c0:c0 + len(part)],
                                   [p[1] for p in part], [p[2] for p in part])
        ctx.pool_size()
    ctx.close()
    total, per_kernel = 0.0, {}
    for ev in prof.key_averages():
        if "k_win_" in ev.key:
            us = ev.self_device_time_total if hasattr(ev, "self_device_time_total") else ev.self_cuda_time_total
            per_kernel[ev.key.split("(")[0]] = {"us_total": us, "launches": ev.count}
            total += us
    steps = sum(1 for _, r, a in lists if r or a)
    return total / 1e3 / max(steps, 1), steps, per_kernel


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"unavailable ({e})"
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this script measures on the device only")
    fr = [synth.make_frame(CAM, 3000 + t, synth.pose_stream(t)) for t in range(N_IMG)]
    G = torch.from_numpy(np.stack([f[0] for f in fr])).pin_memory().numpy()
    D = torch.from_numpy(np.stack([f[1] for f in fr])).pin_memory().numpy()
    P = np.stack([capi.pose16(synth.pose_stream(t)) for t in range(a.frames)])
    results = [dict(gpu_info(), kind="device")]
    modes = [("per_call", 1), ("window_n1", 1), ("window_n8", 8), ("window_n16", 16)]
    for window in (3, 10):
        lists = window_lists(a.frames, window)
        times, ends = {m: [] for m, _ in modes}, {}
        for _ in range(a.rounds):
            for m, k in modes:  # alternating: the modes share whatever else the host and GPU are doing
                ms, *ends[m] = run(m, k, lists, G, D, P)
                times[m].append(ms)
        for m, _ in modes:
            results.append({"window": window, "mode": m, "ms_per_frame_median": float(np.median(times[m])),
                            "ms_per_frame_runs": [round(x, 4) for x in times[m]], "frames_per_s": 1e3 / float(np.median(times[m])),
                            "pool_surfels_at_end": ends[m][0], "stored_surfels_at_end": ends[m][1], "stored_poses_at_end": ends[m][2]})
        ms_step, steps, per_kernel = window_kernel_ms(lists, G, D, P)
        results.append({"window": window, "mode": "window_step_kernels", "ms_per_window_step": ms_step,
                        "frames_with_a_window_step": steps, "kernels": per_kernel})
    for r in results:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
