"""The node's raw and neighbourhood cloud publishers (surfel_map.cpp:1115-1151, :1283-1383), CPU side.

publish_raw_pointcloud is restated in numpy (oracle/pyoracle_clouds.py::raw_cloud): pinned by CRC32s minted from the
reference's own publisher (tests/golden/raw_cloud_checksums.json, tests/golden/make_golden_clouds.py) and, where the
reference node is built, compared with it byte for byte.  publish_neighbor_pointcloud is pinned as "live local points,
then the inactive_pointcloud slice of every BFS pose that is not local", the semantics dsm_pool_export_cloud(ctx, 1)
+ dsm_inactive_export_poses implement.  The device side is tests/test_gpu_node_clouds.py."""
import json
import os

import numpy as np
import pytest

import pyoracle
import pyoracle_clouds
from densesurfelmapping_b200 import synth
from node_drive import build_adapter
from util import CAM, GOLD, canon_points, crc, needs_refmap_clouds, neighbor_replay


def raw_cases():
    """name -> (camera, gray, depth, pose7): quarter-VGA with the synthetic holes, KITTI 1226x370, and a quaternion that
    is neither normalised nor has qw > 0."""
    def frame(cam, t):
        pose = synth.pose_stream(t)
        g, d = synth.make_frame(cam, 700 + t, pose)
        return g, d, pyoracle.pose_to_ros7(pose)
    g0, d0, p0 = frame(CAM, 3)
    g1, d1, p1 = frame(synth.KITTI, 5)
    g2, d2, _ = frame(CAM, 9)
    assert (d0 == 0).sum() > 1000 and (d1 == 0).sum() > 1000
    return {"qvga_holes": (CAM, g0, d0, p0),
            "kitti": (synth.KITTI, g1, d1, p1),
            "qvga_quaternion_qw_negative": (CAM, g2, d2, np.array([1.5, -0.25, 3.0, 0.3, -0.2, 0.1, -0.9]))}


def golden_raw():
    return json.load(open(os.path.join(GOLD, "raw_cloud_checksums.json")))


@pytest.mark.parametrize("case", ["qvga_holes", "kitti", "qvga_quaternion_qw_negative"])
def test_raw_cloud_restatement_is_pinned(case):
    cam, gray, depth, p7 = raw_cases()[case]
    got = pyoracle_clouds.raw_cloud(cam, gray, depth, p7)
    assert got.shape == (cam.width * cam.height, 4)
    # column-major: point i*H + j is column i, row j; a hole lands on T
    i, j = 17, 5
    assert got[i * cam.height + j, 3] == gray[j, i]
    hole = np.argwhere(depth.T.reshape(-1) == 0)[0, 0]
    assert (got[hole, :3] == np.asarray(p7[:3], np.float32)).all()
    assert crc(canon_points(got)) == golden_raw()[case]
    if pyoracle_clouds.have_refmap_clouds():
        m = pyoracle_clouds.RefMapClouds(cam)
        assert m.publish_raw(gray, depth, p7).tobytes() == got.tobytes()
        m.close()


def find_slice(cloud, part):
    """start of `part` as a contiguous run of `cloud` (byte compare), or -1"""
    if len(part) == 0:
        return 0
    starts = np.nonzero((cloud == part[0]).all(1))[0]
    for s in starts:
        if s + len(part) <= len(cloud) and cloud[s:s + len(part)].tobytes() == part.tobytes():
            return int(s)
    return -1


@needs_refmap_clouds
def test_neighbor_pointcloud_is_live_points_then_bfs_slices():
    m = pyoracle_clouds.RefMapClouds(CAM, drift_free_poses=1)
    seen_loop = seen_both = False
    for s in neighbor_replay(m):
        local, inactive = m.local(), m.inactive_points()
        want = [pyoracle.cloud_points(local, 1)]                        # update_times != 0   (:1291-1301)
        for p in s["bfs"]:
            if p in s["window"]:                                       # local pose: skipped (:1311-1312)
                continue
            part = pyoracle.cloud_points(m.attached(p), -(2 ** 31))    # its slice of inactive_pointcloud (:1313-1320)
            assert find_slice(inactive, part) >= 0, f"step {s['t']}: pose {p} is not a slice of inactive_pointcloud"
            want.append(part)
        assert s["published"].tobytes() == np.concatenate(want).tobytes(), f"step {s['t']}"
        seen_loop |= s["t"] == 5 and 0 in s["bfs"] and len(m.attached(0)) > 0
        seen_both |= len(want[0]) > 0 and sum(len(w) for w in want[1:]) > 0
    assert seen_loop and seen_both
    m.close()


def test_node_clouds_helper_compiles_and_fails_loudly_without_gpu(tmp_path):
    import torch
    exe = build_adapter("node_clouds_main")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_gpu_node_clouds.py")
    import subprocess
    cam = CAM
    args = [exe, str(cam.width), str(cam.height)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]
    r = subprocess.run(args + [str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "no usable CUDA device" in r.stderr
