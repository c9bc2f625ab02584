"""Measure dsm::SurfelMapNode (include/dsm_surfel_node.hpp) against the reference node over the product
(oracle/_ref/libdsm_refmap_b200.so: the reference's SurfelMap, the product's fuse kernels) on one drive.

Drive: 1226x370 synthetic frames (8 distinct ones, cycled), --frames frames (>= 300), a keyframe every 4 frames
referenced to the newest keyframe, drift_free_poses 10, and every 100 frames a loop closure whose path moves every pose.
Reported, with the card's name and power limit read in the same run:
  node_ms_per_frame          pose, image and depth callbacks of a frame without a loop closure, device synchronised
  node_publish_ms_per_frame  the active + inactive clouds of every frame, as the reference publishes them
  node_ms_per_loop_event / transforms_per_event   the pose callback of a loop closure and the transforms it enqueued
  inactive_points_ms         one inactive_points() at the drive's final store size
  reference_ms_per_frame     the reference node over the product, all three callbacks (its publishing included)
Usage: python tools/measure_node.py [--frames 320] [--out DIR]"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import synth  # noqa: E402
from test_surfel_node import correction, ros7  # noqa: E402

CAM = synth.KITTI
K = 8


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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to measure on")
    name, power = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return name, power


def run_node(tmp, frames, msgs, publish):
    exe = os.path.join(tmp, "measure_node")
    if not os.path.exists(exe):
        pkg = os.path.join(ROOT, "densesurfelmapping_b200")
        subprocess.run(["g++", "-std=c++11", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tools", "measure_node.cpp"),
                        "-o", exe, "-L", pkg, "-ldsm_b200", f"-Wl,-rpath,{pkg}"], check=True)
    ff, fs = os.path.join(tmp, "frames.bin"), os.path.join(tmp, "script.bin")
    with open(ff, "wb") as f:
        f.write(struct.pack("<i", K))
        for g, d in frames:
            f.write(g.tobytes() + d.tobytes())
    with open(fs, "wb") as f:
        f.write(struct.pack("<i", len(msgs)))
        for t, (stamp, is_kf, ref, p7, path) in enumerate(msgs):
            f.write(struct.pack("<diii", stamp, int(is_kf), ref, t % K) + p7.tobytes())
            f.write(struct.pack("<i", len(path)) + np.asarray(path, np.float64).tobytes() + struct.pack("<ii", 0, int(publish)))
    args = [exe, str(CAM.width), str(CAM.height)] + [repr(float(v)) for v in (CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.far, CAM.near)]
    r = subprocess.run(args + ["10", ff, fs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"measure_node exited {r.returncode}: {r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def run_reference(frames, msgs):
    import pyoracle
    m = pyoracle.RefMap(CAM, drift_free_poses=10, b200=True)
    times = []
    for t, (stamp, is_kf, ref, p7, path) in enumerate(msgs):
        g, d = frames[t % K]
        a = time.perf_counter()
        m.frame(stamp, g, d, p7, is_kf, ref, path7=np.array(path).reshape(-1, 7))
        times.append((time.perf_counter() - a) * 1e3)
    m.close()
    loop = [t for t in range(len(msgs)) if t and t % 100 == 0]
    steady = [x for t, x in enumerate(times) if t not in loop and t >= K]
    return float(np.mean(steady)), [times[t] for t in loop]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert a.frames >= 300
    name, power = card()
    frames = [synth.make_frame(CAM, 5000 + k, synth.pose_stream(k)) for k in range(K)]
    msgs = messages(a.frames)
    with tempfile.TemporaryDirectory() as tmp:
        bare = run_node(tmp, frames, msgs, publish=False)
        pub = run_node(tmp, frames, msgs, publish=True)
    ref_ms, ref_loop = run_reference(frames, msgs)
    res = {"card": name, "power_limit": power, "frames": a.frames, "width": CAM.width, "height": CAM.height,
           "node_ms_per_frame": bare["frame_ms"], "node_publish_ms_per_frame": pub["publish_ms_per_frame"],
           "node_ms_per_loop_event": bare["loop_ms_per_event"], "loop_events": bare["loop_events"],
           "transforms_per_event": bare["transforms"] / max(bare["loop_events"], 1),
           "store_surfels": bare["store_surfels"], "inactive_points_ms": bare["inactive_points_ms"],
           "node_total_ms": bare["total_ms"], "node_with_publish_total_ms": pub["total_ms"],
           "reference_ms_per_frame": ref_ms, "reference_ms_loop_frames": ref_loop}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_node.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
