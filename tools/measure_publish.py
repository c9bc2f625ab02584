"""Measure publishing the node's clouds from inside the stream (dsm_publish_*) against the synchronous readers.

1. The drive of tools/measure_node.py (1226x370, --frames frames, a keyframe every 4, drift_free_poses 10, a loop closure
   every 100 frames) through dsm::SurfelMapNode (tools/measure_publish.cpp) in four modes, alternating on fresh nodes,
   --rounds rounds; ms per frame = host time of the whole drive, the device synchronised at its end, over its frames:
     a  no publishing                         b  active_points() + inactive_points() after every frame
     c  published_clouds() after every fuse   d  published_clouds() of frame t-1 at the start of frame t
   Before the timed rounds every publishing mode runs once with hashing on: the 64-bit hash over every frame's two
   clouds (sizes and bytes) must be the same for b, c and d.
2. A large store through the C ABI (--large surfels, one segment): per snapshot, dsm_pool_export_cloud +
   dsm_inactive_export_cloud against dsm_publish_enqueue + dsm_publish_wait with the store unchanged, host clock.
3. k_cloud_mirror alone (torch.profiler, CUDA activities, --launches launches) at each --sizes store size: with the
   store unchanged, and after a transform of the stored pose (every chunk forwarded).  Bytes by the kernel's model,
   60 N + 32 N_changed; share of the data sheet's 3.35 TB/s HBM3 for the unchanged case; the forwarded case moves
   16 N_changed bytes over PCIe, which bounds it, and is reported as GB/s over PCIe.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_publish.py [--frames 320] [--rounds 3] [--out DIR]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import synth  # noqa: E402
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE  # noqa: E402

CAM = synth.KITTI
SMALL = synth.Camera(320, 240, 262.5, 262.5, 159.5, 119.5, 0.5, 30.0)
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
MODES = "abcd"


def mirror_bytes(n, n_changed):
    """k_cloud_mirror: 44 B surfel + 16 B shadow read per stored surfel, 16 B shadow + 16 B mirror written per forwarded point."""
    return 60 * n + 32 * n_changed


def build_driver(tmp):
    exe = os.path.join(tmp, "measure_publish")
    pkg = os.path.join(ROOT, "densesurfelmapping_b200")
    subprocess.run(["g++", "-std=c++11", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tools", "measure_publish.cpp"),
                    "-o", exe, "-L", pkg, "-ldsm_b200", f"-Wl,-rpath,{pkg}"], check=True)
    return exe


def write_drive(tmp, n_frames):
    import struct
    from measure_node import K, messages
    frames = [synth.make_frame(CAM, 5000 + k, synth.pose_stream(k)) for k in range(K)]
    ff, fs = os.path.join(tmp, "frames.bin"), os.path.join(tmp, "script.bin")
    with open(ff, "wb") as f:
        f.write(struct.pack("<i", K))
        for g, d in frames:
            f.write(g.tobytes() + d.tobytes())
    msgs = messages(n_frames)
    with open(fs, "wb") as f:
        f.write(struct.pack("<i", len(msgs)))
        for t, (stamp, is_kf, ref, p7, path) in enumerate(msgs):
            f.write(struct.pack("<diii", stamp, int(is_kf), ref, t % K) + p7.tobytes())
            f.write(struct.pack("<i", len(path)) + np.asarray(path, np.float64).tobytes() + struct.pack("<ii", 0, 0))
    return ff, fs


def run_mode(exe, ff, fs, mode, check):
    args = [exe, str(CAM.width), str(CAM.height)] + [repr(float(v)) for v in (CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.far, CAM.near)]
    r = subprocess.run(args + ["10", ff, fs, mode, str(int(check))], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"measure_publish mode {mode} exited {r.returncode}: {r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs))}


def node_drive(n_frames, rounds):
    with tempfile.TemporaryDirectory() as tmp:
        exe = build_driver(tmp)
        ff, fs = write_drive(tmp, n_frames)
        checked = {m: run_mode(exe, ff, fs, m, True) for m in "bcd"}
        hashes = {m: r["hash"] for m, r in checked.items()}
        if len(set(hashes.values())) != 1:
            raise RuntimeError(f"the modes published different clouds: {hashes}")
        times = {m: [] for m in MODES}
        last = {}
        for _ in range(rounds):
            for m in MODES:
                last[m] = run_mode(exe, ff, fs, m, False)
                times[m].append(last[m]["ms_per_frame"])
    return {"frames": n_frames, "rounds": rounds, "clouds_hash": hashes["b"], "store_surfels": last["a"]["store_surfels"],
            "pool_surfels": last["a"]["pool_surfels"],
            "inactive_points_at_or_above_changed_from_per_frame": checked["c"]["inactive_points_from_changed_from"] / n_frames,
            "ms_per_frame": {m: spread(times[m]) for m in MODES}}


def stored_context(n, stream=None):
    """A context whose store holds n surfels as one segment (keyframe 0), its pool empty, publishing enabled."""
    from densesurfelmapping_b200 import capi
    ctx = capi.Context(SMALL, max_batch=1, max_local_surfels=max(n, 1 << 16), cuda_stream=stream)
    rng = np.random.default_rng(7)
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz", "nx", "ny", "nz", "color"):
        s[f] = rng.normal(size=n).astype(np.float32)
    s["size"], s["weight"], s["update_times"], s["last_update"] = 0.1, 1.0, 7, 0
    ctx.pool_upload(s)
    ctx.inactive_reserve(n)
    assert ctx.inactive_retire(0) == n
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.publish_enable()
    return ctx


def warp():
    a = np.deg2rad(0.5)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    Wm[:3, 3] = [0.01, -0.02, 0.005]
    return Wm


def large_store(n, reps, rounds):
    ctx = stored_context(n)
    lib, h = ctx.lib, ctx.h
    out = np.zeros(n + 1, POINT_DTYPE)
    got = ctypes.c_int(0)
    act = np.zeros(1, POINT_DTYPE)
    ctx.publish_enqueue(5)
    _, first, _ = ctx.publish_wait()
    if first.tobytes() != ctx.inactive_export_cloud().tobytes():
        raise RuntimeError("the published inactive cloud differs from dsm_inactive_export_cloud")

    def readers():
        assert lib.dsm_pool_export_cloud(h, 5, act.ctypes.data, 0, ctypes.byref(got)) == 0
        assert lib.dsm_inactive_export_cloud(h, out.ctypes.data, n, ctypes.byref(got)) == 0

    def published():
        assert lib.dsm_publish_enqueue(h, 5) == 0
        assert lib.dsm_publish_wait(h, None, None, None, None, None) == 0

    times = {"readers": [], "published": []}
    for fn in (readers, published):
        fn()
    for _ in range(rounds):
        for name, fn in (("readers", readers), ("published", published)):
            ctx.sync()
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            ctx.sync()
            times[name].append((time.perf_counter() - t0) * 1e3 / reps)
    ctx.close()
    return {"store_surfels": n, "snapshots_per_round": reps, "rounds": rounds,
            "ms_per_snapshot": {k: spread(v) for k, v in times.items()}}


def kernel_alone(n, launches):
    import torch
    from torch.profiler import ProfilerActivity, profile
    ctx = stored_context(n)
    lib, h = ctx.lib, ctx.h
    ctx.publish_enqueue(5)
    ctx.publish_wait()
    res = {"store_surfels": n, "launches": launches}
    for case in ("unchanged", "all_forwarded"):
        def step():
            if case == "all_forwarded":
                ctx.inactive_transform(0, warp())
            assert lib.dsm_publish_enqueue(h, 5) == 0
            assert lib.dsm_publish_wait(h, None, None, None, None, None) == 0
        for _ in range(5):
            step()
        n_chunks = ctx.publish_chunks()
        changed = min(n, n_chunks * 256)
        if (case == "unchanged") != (n_chunks == 0):
            raise RuntimeError(f"{case}: {n_chunks} chunks forwarded")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(launches):
                step()
            ctx.sync()
            torch.cuda.synchronize()
        rows = [k for k in prof.key_averages() if "k_cloud_mirror" in k.key]
        count = sum(k.count for k in rows)
        total_us = sum(getattr(k, "device_time_total", None) or getattr(k, "cuda_time_total") for k in rows)
        if count != launches:
            raise RuntimeError(f"profiler saw {count} launches of k_cloud_mirror, expected {launches}")
        us = total_us / count
        nbytes = mirror_bytes(n, changed)
        r = {"us": us, "model_bytes": nbytes, "model_GBps": nbytes / us * 1e-3, "chunks_forwarded": n_chunks}
        if case == "unchanged":
            r["bound"] = "HBM"
            r["share_of_3.35TBps"] = nbytes / (us * 1e-6) / HBM_BYTES_PER_S
        else:
            r["bound"] = "PCIe"
            r["pcie_GBps"] = 16 * changed / us * 1e-3
        res[case] = r
    ctx.close()
    return res


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        r = None
    if r is None or r.returncode != 0 or not r.stdout.strip():
        raise RuntimeError("nvidia-smi failed: no GPU to measure on")
    name, power = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--large", type=int, default=1 << 20, help="stored surfels of the large-store comparison")
    ap.add_argument("--sizes", type=int, nargs="+", default=[46700, 1 << 20, 1 << 22], help="store sizes of the kernel timing")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true", help="build the driver and write the drive, then stop (no GPU needed)")
    a = ap.parse_args()
    if a.launches < 200 and not a.dry_run:
        ap.error("--launches must be at least 200")
    if a.dry_run:
        with tempfile.TemporaryDirectory() as tmp:
            build_driver(tmp)
            ff, fs = write_drive(tmp, a.frames)
            print(json.dumps({"dry_run": True, "frames_bytes": os.path.getsize(ff), "script_bytes": os.path.getsize(fs),
                              "model_bytes_1Mi_unchanged": mirror_bytes(1 << 20, 0)}))
        return
    name, power = card()
    res = {"card": name, "power_limit": power, "width": CAM.width, "height": CAM.height}
    res["node_drive"] = node_drive(a.frames, a.rounds)
    res["large_store"] = large_store(a.large, 20, a.rounds)
    res["k_cloud_mirror"] = [kernel_alone(n, a.launches) for n in a.sizes]
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_publish.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
