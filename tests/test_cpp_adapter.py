"""The C++ drop-in: include/dsm_fusion_functions.hpp mirrors the reference's FusionFunctions class.
CPU: it compiles against cv::Mat / Eigen-like caller types and links to the C ABI; without a GPU it
fails loudly (exit code 3, no fallback).  GPU: its results match the oracle."""
import os
import struct
import subprocess

import numpy as np
import pytest

from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from node_drive import build_adapter, cam_args


def run_adapter(tmp, cam, ref, pose, gray, depth, local):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<i", ref) + np.asarray(pose, np.float32).tobytes() + struct.pack("<i", len(local)))
        f.write(gray.tobytes() + depth.tobytes() + local.tobytes())
    args = [build_adapter()] + cam_args(cam) + [fin, fout]
    r = subprocess.run(args, capture_output=True, text=True)
    return r, fout


def test_adapter_compiles_and_fails_loudly_without_gpu(tmp_path):
    import torch
    build_adapter()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    cam = synth.VGA
    g, d = synth.make_frame(cam, 0)
    r, _ = run_adapter(str(tmp_path), cam, 0, synth.identity_pose(), g, d, np.zeros(0, SURFEL_DTYPE))
    assert r.returncode == 3 and "no usable CUDA device" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    from util import check_surfels, oracle_for
    build_adapter()
    cam = synth.VGA
    g, d = synth.make_frame(cam, 0)
    pose = synth.identity_pose()
    orc = oracle_for(cam)
    _, pool = orc.fuse(0, g, d, pose, np.zeros(0, SURFEL_DTYPE))
    want_local, want_new = orc.fuse(1, g, d, pose, pool)
    r, fout = run_adapter(str(tmp_path), cam, 1, pose, g, d, pool)
    assert r.returncode == 0, r.stderr
    raw = open(fout, "rb").read()
    nl = struct.unpack_from("<i", raw, 0)[0]
    local = np.frombuffer(raw, SURFEL_DTYPE, nl, 4)
    nn = struct.unpack_from("<i", raw, 4 + 44 * nl)[0]
    new = np.frombuffer(raw, SURFEL_DTYPE, nn, 8 + 44 * nl)
    check_surfels(local, want_local, "adapter local")
    check_surfels(new, want_new, "adapter new")


# ---- include/dsm_surfel_map.hpp: the SurfelMap-side helper for the GPU-resident pool (INTEGRATION.md §4) ----
def write_stream(path, cam, frames, warp, retire_kf):
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(frames)))
        for ref, pose, gray, depth in frames:
            f.write(struct.pack("<i", ref) + np.asarray(pose, np.float32).tobytes() + gray.tobytes() + depth.tobytes())
        f.write(np.asarray(warp, np.float32).tobytes() + struct.pack("<i", retire_kf))


def run_resident(tmp, cam, frames, warp, retire_kf):
    exe = build_adapter("resident_main")
    fin = os.path.join(tmp, "stream.bin")
    outs = [os.path.join(tmp, n) for n in ("out.bin", "cloud.pcd", "mesh.ply")]
    write_stream(fin, cam, frames, warp, retire_kf)
    args = [exe] + cam_args(cam) + [fin] + outs
    return subprocess.run(args, capture_output=True, text=True), outs


def test_resident_helper_compiles_and_fails_loudly_without_gpu(tmp_path):
    import torch
    build_adapter("resident_main")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    cam = synth.VGA
    g, d = synth.make_frame(cam, 0)
    r, _ = run_resident(str(tmp_path), cam, [(0, synth.identity_pose(), g, d)], synth.identity_pose(), 0)
    assert r.returncode == 3 and "no usable CUDA device" in r.stderr


@pytest.mark.gpu
def test_resident_helper_flow_matches_oracle(tmp_path):
    import pyoracle
    from util import oracle_for
    cam = synth.VGA
    orc = oracle_for(cam)
    frames, pool = [], np.zeros(0, SURFEL_DTYPE)
    for t in range(3):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 800 + t, pose)
        frames.append((t, pose, gray, depth))
        lo, no = orc.fuse(t, gray, depth, pose, pool)
        pool = pyoracle.fuse_map_poststep(lo, no)
    a = np.deg2rad(1.0)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    Wm[:3, 3] = [0.2, 0.0, -0.1]
    w = np.ascontiguousarray(Wm.T.astype(np.float32).reshape(16))
    r, (fout, fpcd, fply) = run_resident(str(tmp_path), cam, frames, w, 1)
    assert r.returncode == 0, r.stderr
    raw, arrs, o = open(fout, "rb").read(), [], 0
    for dt in (SURFEL_DTYPE, SURFEL_DTYPE, SURFEL_DTYPE, np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4")])):
        n = struct.unpack_from("<i", raw, o)[0]
        arrs.append(np.frombuffer(raw, dt, n, o + 4))
        o += 4 + n * dt.itemsize
    got_pool, retired, final_pool, points = arrs
    assert abs(len(got_pool) - len(pool)) <= max(2, len(pool) // 500)   # free-running stream (see test_gpu_resident)
    # everything after the stream is exact bookkeeping on got_pool
    warped = pyoracle.warp_active(got_pool, w)
    want_local, want_out = pyoracle.retire(warped, 1)
    from util import check_surfels
    check_surfels(retired, want_out, "retired")
    want_final = np.concatenate([want_local, want_out])
    check_surfels(final_pool, want_final, "final pool")
    want_pts = pyoracle.cloud_points(final_pool, 5)
    assert points.tobytes() == want_pts.tobytes()
    assert open(fpcd).read() == pyoracle.pcd_text(want_pts)
    assert open(fply).read() == pyoracle.ply_mesh_text(np.concatenate([retired, final_pool[final_pool["update_times"] >= 5]]))
