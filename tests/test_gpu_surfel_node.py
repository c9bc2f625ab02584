"""dsm::SurfelMapNode on the GPU (tests/cpp/node_main.cpp) against the reference's own SurfelMap over the product
(pyoracle_window.RefMapWindow(b200=True): its move_add_surfels, warp_surfels and host post-step, the product's fuse
kernels).  After every message: local_surfels slot for slot, every pose's attached_surfels and the published clouds
byte for byte, except the points the reference leaves stale after a loop closure; at the end the save_mesh PLY byte for
byte and the save_cloud PCD except those points.  Drives: tests/test_surfel_node.drive (loop paths that move every pose,
a path shorter than the pose database, keyframe 0 brought back by a loop edge, keyframes retired, reactivated and
retired again)."""
import os

import numpy as np
import pytest

import pyoracle
import pyoracle_window
from densesurfelmapping_b200 import capi, synth
from test_surfel_node import Script, drive, read_dumps, run_node

pytestmark = pytest.mark.gpu
needs_b200_node = pytest.mark.skipif(not pyoracle_window.have_refmap_window(b200=True),
                                     reason="oracle/_ref/libdsm_refmap_window_b200.so not built")
N_FRAMES = 30


def frames(cam, n=N_FRAMES):
    return [synth.make_frame(cam, 3000 + t, synth.pose_stream(t)) for t in range(n)]


def points_of(surfels):
    return np.stack([surfels["px"], surfels["py"], surfels["pz"], surfels["color"]], -1).astype(np.float32).reshape(-1, 4)


class Stale:
    """The reference's stale inactive points: after warp_surfels, the last point of a warped pose's slice of
    inactive_pointcloud keeps its value from before the first warp since the pose's retirement (surfel_map.cpp:742)."""

    def __init__(self):
        self.pre = {}   # pose -> its last point before the first warp since retirement

    def warped(self, poses, attached_before):
        for p in poses:
            if len(attached_before[p]) and p not in self.pre:
                self.pre[p] = points_of(attached_before[p][-1:])[0]

    def moved(self, poses):   # retired afresh or reactivated: a new slice, or none
        for p in poses:
            self.pre.pop(p, None)

    def check(self, got, want, attached, what):
        """got (node) equals want (reference) except at rows where the reference holds a stale pose's pre-warp point
        and the node that pose's current last point; returns the number of such rows."""
        got = got.view(np.float32).reshape(-1, 4)
        assert got.shape == want.shape, f"{what}: {len(got)} != {len(want)} points"
        bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))[0]
        for i in bad:
            ok = any(want[i].tobytes() == pre.tobytes() and got[i].tobytes() == points_of(attached[p][-1:])[0].tobytes()
                     for p, pre in self.pre.items())
            assert ok, f"{what}: point {i} differs ({got[i]} vs {want[i]}) and is not a stale point"
        return len(bad)


def compare_map(d, m, ref, stale, what):
    assert d["map_rc"] == 0, what
    assert d["local_surfels"].tobytes() == m.local().tobytes(), f"{what}: local_surfels"
    for p in range(m.num_poses()):
        assert d["attached"][p].tobytes() == m.attached(p).tobytes(), f"{what}: attached_surfels of pose {p}"
    m.publish_clouds(ref)
    assert d["active"].tobytes() == m.published("active_pointcloud").tobytes(), f"{what}: active cloud"
    n = stale.check(d["inactive"], m.published("inactive_pointcloud"), d["attached"], f"{what}: inactive cloud")
    assert n == sum(1 for p, pre in stale.pre.items() if pre.tobytes() != points_of(d["attached"][p][-1:])[0].tobytes())
    stale.check(d["all"], m.published("pointcloud"), d["attached"], f"{what}: all cloud")
    stale.check(d["neighbor"], m.published("neighbor_pointcloud"), d["attached"], f"{what}: neighbour cloud")
    return n


def node_script(msgs, frs, tmp):
    sc = Script()
    for (stamp, is_kf, ref, p7, path, loops), (gray, depth) in zip(msgs, frs):
        sc.orb(stamp, is_kf, ref, p7, path, loops)
        sc.dump(True, True, ref)
        sc.images(stamp, gray, depth)
        sc.dump(True, True, ref)
    sc.save(os.path.join(tmp, "node.ply"), os.path.join(tmp, "node.pcd"))
    return sc


@needs_b200_node
@pytest.mark.parametrize("drift_free_poses", [1, 2, 10])
def test_node_equals_the_reference_node_over_the_product(tmp_path, drift_free_poses):
    cam = synth.KITTI
    msgs, frs = drive(N_FRAMES), frames(cam)
    _, raw = run_node(str(tmp_path), cam, node_script(msgs, frs, str(tmp_path)), drift_free_poses, device=0)
    dumps = iter(read_dumps(raw, [(True, True)] * (2 * N_FRAMES)))
    m = pyoracle_window.RefMapWindow(cam, drift_free_poses=drift_free_poses, b200=True)
    stale, prev, n_stale, n_warps = Stale(), None, 0, 0
    for t, ((stamp, is_kf, ref, p7, path, loops), (gray, depth)) in enumerate(zip(msgs, frs)):
        m.frame(stamp, None, None, p7, is_kf, ref, path7=np.array(path).reshape(-1, 7), loops=loops)
        d = next(dumps)
        assert d["rc"] == 0
        if d["warp"]:
            n_warps += 1
            stale.warped([p for p, _ in d["warp"][1:]], prev["attached"] if prev else [])
        n_stale = max(n_stale, compare_map(d, m, ref, stale, f"frame {t} after its pose"))
        pending = m.pending_frame()
        assert d["pending"][0] == pending[0] and d["pending"][1].tobytes() == pending[1].tobytes()
        m.images(stamp, gray, depth)
        stale.moved(pending[2] + pending[3])
        prev = next(dumps)
        assert prev["rc"] == 0
        compare_map(prev, m, ref, stale, f"frame {t} after its fuse")
    assert n_warps >= 2
    if drift_free_poses <= 2:
        assert n_stale > 0, "no stale point was exercised"
    # save_mesh: every pose's attached surfels in index order, then the local ones: byte for byte
    m.save_mesh(str(tmp_path / "ref.ply"))
    assert open(tmp_path / "node.ply", "rb").read() == open(tmp_path / "ref.ply", "rb").read()
    # save_cloud: the PCD of the node's cloud, which is the reference's except its stale points
    cloud = m.save_cloud(str(tmp_path / "ref.pcd"))
    stale.check(prev["all"], cloud, prev["attached"], "save_cloud")
    assert open(tmp_path / "node.pcd").read() == pyoracle.pcd_text(prev["all"].view(np.float32).reshape(-1, 4))
    m.close()


@pytest.mark.skipif(not pyoracle_window.have_refmap_window(), reason="oracle/_ref/libdsm_refmap_window.so not built")
def test_rgbd_constants_at_720p(tmp_path):
    """The RGBD constant set at 1280x720: the node equals the per-call entry points (dsm_pool_transform,
    dsm_inactive_transform, dsm_inactive_retire / _reactivate, dsm_fuse_frame_resident) run with RGBD constants on the
    fuse poses, window lists and warp matrices the node used, which the CPU tests pin to the reference node."""
    cam, n = synth.HD, 24
    msgs, frs = drive(n), frames(cam, n)
    _, raw = run_node(str(tmp_path), cam, node_script(msgs, frs, str(tmp_path)), 2, device=0, rgbd=True)
    dumps = iter(read_dumps(raw, [(True, True)] * (2 * n)))
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=1 << 20)
    ctx.set_constants(capi.CONSTANTS_RGBD)
    ctx.pool_upload(np.zeros(0, pyoracle.SURFEL_DTYPE))
    ctx.inactive_reserve(1 << 21)

    def same(d, what):
        assert d["map_rc"] == 0, what
        assert d["local_surfels"].tobytes() == ctx.pool_download().tobytes(), f"{what}: local_surfels"
        for p in range(len(d["cam"])):
            assert d["attached"][p].tobytes() == ctx.inactive_download(p).tobytes(), f"{what}: pose {p}"
        assert d["inactive"].tobytes() == ctx.inactive_export_cloud().tobytes(), f"{what}: inactive cloud"

    warps = 0
    for t, (gray, depth) in enumerate(frs):
        d = next(dumps)
        for p, W in d["warp"]:
            if p < 0:
                ctx.pool_transform(W)
            else:
                ctx.inactive_transform(p, W)
        warps += bool(d["warp"])
        same(d, f"frame {t} after its pose")
        ref, pose, rem, add = d["pending"]
        for kf in rem:
            ctx.inactive_retire(kf)
        for kf in add:
            ctx.inactive_reactivate(kf)
        ctx.fuse_frame_resident(ref, gray, depth, pose)
        same(next(dumps), f"frame {t} after its fuse")
    assert warps >= 2 and ctx.inactive_size()[0] > 0
    ctx.close()


@needs_b200_node
def test_store_overflow_reported_by_the_next_read(tmp_path):
    """An inactive store too small for the drive: the frame that would overflow it is not applied, the next read returns
    DSM_E_CAPACITY, and the map read after that is the map after the last applied frame."""
    cam, n = synth.KITTI, 10
    msgs, frs = drive(n), frames(cam, n)
    full = Script()
    small = Script()
    for (stamp, is_kf, ref, p7, path, loops), (gray, depth) in zip(msgs, frs):
        for sc in (full, small):
            sc.orb(stamp, is_kf, ref, p7, path, loops)
            sc.images(stamp, gray, depth)
            sc.dump(True, True, ref)
        small.dump(True, True, ref)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    _, raw_full = run_node(str(tmp_path / "a"), cam, full, 1, device=0)
    _, raw_small = run_node(str(tmp_path / "b"), cam, small, 1, device=0, max_inactive=1)
    want = read_dumps(raw_full, [(True, True)] * n)
    got = read_dumps(raw_small, [(True, True)] * (2 * n))
    first = next(t for t in range(n) if got[2 * t]["map_rc"] != 0)
    assert first > 0 and got[2 * first]["map_rc"] == -6
    assert all(got[2 * t]["map_rc"] == 0 and got[2 * t]["local_surfels"].tobytes() == want[t]["local_surfels"].tobytes()
               for t in range(first))
    after = got[2 * first + 1]
    assert after["map_rc"] == 0
    assert after["local_surfels"].tobytes() == want[first - 1]["local_surfels"].tobytes()
    assert after["inactive"].tobytes() == want[first - 1]["inactive"].tobytes()
