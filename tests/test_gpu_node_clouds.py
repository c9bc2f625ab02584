"""dsm_frame_raw_cloud and dsm_inactive_export_poses on the H100: the node's raw cloud (publish_raw_pointcloud,
surfel_map.cpp:1115-1151) byte-identical to the numpy restatement the CPU suite pins against the reference, from the
frame slots of every entry point that takes images; the neighbourhood cloud (publish_neighbor_pointcloud, :1283-1383)
byte-identical to the reference node's in a controlled replay; and the C++ helper's neighbor_points / raw_points."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

import pyoracle_clouds
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from test_cpp_adapter import build_adapter
from test_node_clouds import CAM, canon_points, needs_refmap_clouds, neighbor_replay

pytestmark = pytest.mark.gpu

P7 = np.array([0.4, -1.25, 2.5, 0.12, -0.31, 0.05, -0.93])  # not normalised, qw < 0


def frames(cam, n, seed):
    out = []
    for t in range(n):
        pose = synth.pose_stream(seed + t)
        g, d = synth.make_frame(cam, seed + t, pose)
        out.append((pose, g, d))
    return out


def check_raw(ctx, frame, cam, gray, depth, what):
    got = ctx.frame_raw_cloud(frame, P7)
    want = pyoracle_clouds.raw_cloud(cam, gray, depth, P7)
    assert got.dtype == POINT_DTYPE and len(got) == cam.width * cam.height, what
    got = got.view(np.float32).reshape(-1, 4)
    assert canon_points(got) == canon_points(want), f"{what}: {(got != want).any(1).sum()} points differ"


@pytest.mark.parametrize("cam", [synth.VGA, synth.KITTI], ids=["vga", "kitti"])
def test_raw_cloud_after_fuse_frame_resident(cam):
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=200000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for t, (pose, g, d) in enumerate(frames(cam, 3, 40)):   # frame slots 0, 1, 0
        ctx.fuse_frame_resident(t, g, d, pose)
        check_raw(ctx, 0, cam, g, d, f"resident frame {t}")
    ctx.close()


def test_raw_cloud_after_fuse_stream_resident():
    cam = synth.VGA
    ctx = capi.Context(cam, max_batch=8, max_local_surfels=400000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for run in range(2):   # two runs of 4 frames: both halves of the frame slots
        fr = frames(cam, 4, 60 + 4 * run)
        ctx.fuse_stream_resident(np.arange(4) + 4 * run, np.stack([g for _, g, _ in fr]), np.stack([d for _, _, d in fr]),
                                 np.stack([p for p, _, _ in fr]))
        for b, (_, g, d) in enumerate(fr):
            check_raw(ctx, b, cam, g, d, f"stream run {run} frame {b}")
    ctx.close()


def batch_args(cam, n, seed):
    fr = frames(cam, n, seed)
    return (np.arange(n, dtype=np.int32), np.ascontiguousarray(np.stack([g for _, g, _ in fr])),
            np.ascontiguousarray(np.stack([d for _, _, d in fr])), np.ascontiguousarray(np.stack([p for p, _, _ in fr])))


def test_raw_cloud_after_batch_calls():
    cam = synth.KITTI
    n = 4
    ref, g, d, p = batch_args(cam, n, 80)
    ctx = capi.Context(cam, max_batch=n, max_local_surfels=1000)
    L, S = ctx.lib, ctx.S
    ofs = np.zeros(n + 1, np.int32)
    new = np.zeros(n * S, SURFEL_DTYPE)
    cnt = np.zeros(n, np.int32)
    ptrs = (ref.ctypes.data, g.ctypes.data, d.ctypes.data, p.ctypes.data, None, ofs.ctypes.data, new.ctypes.data, cnt.ctypes.data)
    ctx._ck(L.dsm_fuse_batch(ctx.h, n, *ptrs))
    check_raw(ctx, 2, cam, g[2], d[2], "dsm_fuse_batch frame 2")
    # asynchronous batch (two chunks on their own streams), raw cloud asked for before dsm_batch_wait
    ref2, g2, d2, p2 = batch_args(cam, n, 90)
    ctx._ck(L.dsm_fuse_batch_async(ctx.h, n, ref2.ctypes.data, g2.ctypes.data, d2.ctypes.data, p2.ctypes.data, None,
                                   ofs.ctypes.data, new.ctypes.data, cnt.ctypes.data))
    check_raw(ctx, 3, cam, g2[3], d2[3], "dsm_fuse_batch_async frame 3")
    ctx._ck(L.dsm_batch_wait(ctx.h))
    ctx.batch_upload(ref, g, d, p, np.zeros(0, SURFEL_DTYPE), ofs)   # dsm_batch_upload: frames before any run
    check_raw(ctx, 1, cam, g[1], d[1], "dsm_batch_upload frame 1")
    ctx.close()


def test_raw_cloud_after_fuse_frame_with_padded_pitches_and_errors():
    cam = CAM
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=100000)
    L = ctx.lib
    n = ctypes.c_int(-1)
    p7 = np.ascontiguousarray(P7)
    out = np.zeros(cam.width * cam.height, POINT_DTYPE)
    assert L.dsm_frame_raw_cloud(ctx.h, 0, p7.ctypes.data, out.ctypes.data, len(out), ctypes.byref(n)) == -7  # DSM_E_STATE
    pose, g, d = frames(cam, 1, 120)[0]
    gp = np.zeros((cam.height, cam.width + 29), np.uint8)       # padded rows: a 2-D copy into the packed staging
    dp = np.zeros((cam.height, cam.width + 19), np.float32)
    gp[:, :cam.width], dp[:, :cam.width] = g, d
    new = np.zeros(ctx.S, SURFEL_DTYPE)
    pose = np.ascontiguousarray(pose)
    ctx._ck(L.dsm_fuse_frame(ctx.h, 0, gp.ctypes.data, gp.strides[0], dp.ctypes.data, dp.strides[0], pose.ctypes.data, None, 0,
                             new.ctypes.data, ctx.S, ctypes.byref(n)))
    check_raw(ctx, 0, cam, g, d, "dsm_fuse_frame padded")
    want = pyoracle_clouds.raw_cloud(cam, g, d, P7)
    cap = 1000
    part = np.zeros(cap + 8, POINT_DTYPE)
    assert L.dsm_frame_raw_cloud(ctx.h, 0, p7.ctypes.data, part.ctypes.data, cap, ctypes.byref(n)) == 0
    assert n.value == cam.width * cam.height
    assert part[:cap].view(np.float32).reshape(-1, 4).tobytes() == want[:cap].tobytes() and not part[cap:].view(np.float32).any()
    assert L.dsm_frame_raw_cloud(ctx.h, 0, p7.ctypes.data, None, 0, ctypes.byref(n)) == 0 and n.value == cam.width * cam.height
    for frame, pp, o, c in ((1, p7.ctypes.data, out.ctypes.data, len(out)), (-1, p7.ctypes.data, out.ctypes.data, len(out)),
                            (0, None, out.ctypes.data, len(out)), (0, p7.ctypes.data, None, 10), (0, p7.ctypes.data, out.ctypes.data, -1)):
        assert L.dsm_frame_raw_cloud(ctx.h, frame, pp, o, c, ctypes.byref(n)) == -1   # DSM_E_INVALID
    assert L.dsm_frame_raw_cloud(ctx.h, 0, p7.ctypes.data, out.ctypes.data, len(out), None) == -1
    ctx.close()


@needs_refmap_clouds
def test_neighbor_cloud_equals_reference_node():
    """Each step of the CPU suite's replay (tests/test_node_clouds.py::neighbor_replay): the device gets the node's pool
    from before move_add_surfels, retires / reactivates the same poses on its inactive store, and its neighbourhood
    cloud -- dsm_pool_export_cloud(ctx, 1) then dsm_inactive_export_poses(BFS list) -- must equal what the node's
    publish_neighbor_pointcloud sent, byte for byte."""
    m = pyoracle_clouds.RefMapClouds(CAM, drift_free_poses=1)
    ctx = capi.Context(CAM, max_batch=2, max_local_surfels=60000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.inactive_reserve(200000)
    with_inactive = 0
    for s in neighbor_replay(m):
        ctx.pool_upload(s["pool"])
        for p in sorted(set(s["window_before"]) - set(s["window"])):     # move_add_surfels: removal in set order ...
            ctx.inactive_retire(p)
        for p in [q for q in s["bfs"] if q in s["window"] and q not in s["window_before"]]:   # ... then insertion
            ctx.inactive_reactivate(p)
        assert ctx.pool_download().tobytes() == m.local().tobytes(), f"step {s['t']}: pool"
        live = ctx.pool_export_cloud(1).view(np.float32).reshape(-1, 4)
        inact = ctx.inactive_export_poses(s["bfs"]).view(np.float32).reshape(-1, 4)
        got = np.concatenate([live, inact])
        assert got.tobytes() == s["published"].tobytes(), f"step {s['t']}: {len(got)} vs {len(s['published'])} points"
        # the whole store is the node's inactive_pointcloud; cap < total writes a prefix
        assert ctx.inactive_export_cloud().view(np.float32).reshape(-1, 4).tobytes() == m.inactive_points().tobytes()
        if len(inact) > 3:
            assert ctx.inactive_export_poses(s["bfs"], cap=3).view(np.float32).reshape(-1, 4).tobytes() == inact[:3].tobytes()
        with_inactive += len(inact) > 0
    assert with_inactive >= 5
    with pytest.raises(capi.DsmError):
        ctx._ck(ctx.lib.dsm_inactive_export_poses(ctx.h, None, -1, None, 0, ctypes.byref(ctypes.c_int())))
    ctx.close()
    m.close()


def test_node_clouds_cpp_helper(tmp_path):
    cam = CAM
    exe = build_adapter("node_clouds_main")
    fr = frames(cam, 3, 200)
    bfs = [2, 1, 7, 0]   # 2 stays local, 7 does not exist, 1 and 0 are retired (in that order of the store: 0 then 1)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<i", len(fr)))
        for t, (pose, g, d) in enumerate(fr):
            f.write(struct.pack("<i", t) + np.asarray(pose, np.float32).tobytes() + g.tobytes() + d.tobytes())
        f.write(struct.pack("<3i", 0, 1, len(bfs)) + np.asarray(bfs, np.int32).tobytes() + np.asarray(P7, np.float64).tobytes())
    args = [exe, str(cam.width), str(cam.height)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]
    r = subprocess.run(args + [fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw, o, arrs = open(fout, "rb").read(), 0, []
    for k in range(5):
        n = struct.unpack_from("<i", raw, o)[0]
        o += 4
        if k == 3:
            arrs.append(n)
            continue
        arrs.append(np.frombuffer(raw, np.float32, 4 * n, o).reshape(-1, 4))
        o += 16 * n
    neighbor, active1, inactive, n_first, points = arrs
    assert 0 < n_first < len(inactive)
    assert neighbor.tobytes() == np.concatenate([active1, inactive[n_first:], inactive[:n_first]]).tobytes()
    _, g, d = fr[-1]
    assert canon_points(points) == canon_points(pyoracle_clouds.raw_cloud(cam, g, d, P7))
