"""Shared by the node measurements tools/measure_*.py: the card, the spread of repeated runs, the drive their harnesses
read (frames.bin and script.bin, the layout tools/measure_drive.hpp gives) building and running a harness, the profiler's kernel times, and the random maps the checkpoint measurements save.

Drive: 1226x370 synthetic frames (K distinct ones, cycled), a keyframe every 4 frames referenced to the newest keyframe,
and every 100 frames a loop closure whose path moves every pose."""
import json
import os
import struct
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402
from node_drive import cam_args, correction, ros7  # noqa: E402

CAM = synth.KITTI
K = 8
SMALL = synth.Camera(320, 240, 262.5, 262.5, 159.5, 119.5, 0.5, 30.0)   # the contexts the kernels are measured on


def card():
    """(name, power limit) of the card; raises when nvidia-smi is missing or fails."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        r = None
    if r is None or r.returncode != 0 or not r.stdout.strip():
        raise RuntimeError("nvidia-smi failed: no GPU to measure on")
    name, power = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return name, power


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs))}


def images():
    return [synth.make_frame(CAM, 5000 + k, synth.pose_stream(k)) for k in range(K)]


def messages(n_frames):
    out, kf_frames, last_kf = [], [], 0
    for t in range(n_frames):
        C = correction(t // 100)
        P = np.asarray(synth.pose_stream(t), np.float64).reshape(4, 4).T
        is_kf = t % 4 == 0
        path = [ros7(C @ np.asarray(synth.pose_stream(f), np.float64).reshape(4, 4).T) for f in kf_frames]
        out.append((100.0 + 0.1 * t, is_kf, last_kf if t else 0, ros7(C @ P), path))
        if is_kf:
            kf_frames.append(t)
            last_kf = len(kf_frames) - 1
    return out


def write_drive(tmp, imgs, msgs, publish=False):
    """frames.bin and script.bin in tmp; message t shows frame t % K.  publish: the script's per-frame publish flag."""
    ff, fs = os.path.join(tmp, "frames.bin"), os.path.join(tmp, "script.bin")
    with open(ff, "wb") as f:
        f.write(struct.pack("<i", len(imgs)))
        for g, d in imgs:
            f.write(g.tobytes() + d.tobytes())
    with open(fs, "wb") as f:
        f.write(struct.pack("<i", len(msgs)))
        for t, (stamp, is_kf, ref, p7, path) in enumerate(msgs):
            f.write(struct.pack("<diii", stamp, int(is_kf), ref, t % len(imgs)) + p7.tobytes())
            f.write(struct.pack("<i", len(path)) + np.asarray(path, np.float64).tobytes() + struct.pack("<ii", 0, int(publish)))
    return ff, fs


def build_harness(tmp, name):
    """tools/<name>.cpp compiled into tmp."""
    exe = os.path.join(tmp, name)
    pkg = os.path.join(ROOT, "densesurfelmapping_b200")
    subprocess.run(["g++", "-std=c++11", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tools", name + ".cpp"),
                    "-o", exe, "-L", pkg, "-ldsm_b200", f"-Wl,-rpath,{pkg}"], check=True)
    return exe


def run_harness(exe, ff, fs, args=()):
    """The harness on the drive with drift_free_poses 10 and its own arguments; returns the JSON object it prints."""
    r = subprocess.run([exe] + cam_args(CAM) + ["10", ff, fs] + [str(a) for a in args], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{os.path.basename(exe)} {' '.join(map(str, args))} exited {r.returncode}: {r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def kernel_us(fn, names):
    """Per-launch device time in us of each kernel in `names` over what fn() enqueues."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: [] for n in names}
    for e in prof.events():
        for n in names:
            if n in e.name:
                t = getattr(e, "device_time", None)
                out[n].append(float(t if t is not None else e.cuda_time))
    return out


# ---- the maps of the checkpoint measurements ----
SIZES = {"node": (81 << 10, 47 << 10, 80), "large": (1 << 20, 4 << 20, 1024)}


def surfels(rng, n):
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
        s[f] = rng.standard_normal(n).astype(np.float32)
    s["update_times"] = rng.integers(1, 20, n)
    return s


def make_map(n_pool, n_store, n_seg, seed=7):
    rng = np.random.default_rng(seed)
    ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=n_pool)
    ctx.pool_upload(surfels(rng, n_pool))
    ctx.inactive_reserve(n_store)
    store = surfels(rng, n_store)
    cnt = np.full(n_seg, n_store // n_seg, np.int32)
    cnt[-1] += n_store - cnt.sum()
    ofs = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
    store["last_update"] = np.repeat(np.arange(n_seg, dtype=np.int32), cnt)
    ctx.inactive_load(store, np.stack([np.arange(n_seg, dtype=np.int32), ofs, cnt], 1))
    return ctx
