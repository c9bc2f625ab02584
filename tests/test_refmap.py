"""The reference's whole SurfelMap compiled in place (oracle/ref_map_driver.cpp -> oracle/_ref/libdsm_refmap.so).

CPU: (1) the restated SurfelMap members this repo's tests lean on -- fuse_map's post-step, the active-surfel warp,
move_add_surfels' removal loop, the cloud builders -- are pinned against the reference's own code; (2) the PRODUCT's
PLY-mesh writer and hexagon generator (host code in the C ABI) are compared byte for byte with save_mesh /
push_a_surfel of the reference; (3) INTEGRATION.md's three-line patch is shown to compile against the unmodified
surfel_map.cpp (libdsm_refmap_b200.so).  GPU: the same stream through the
reference node with its own FusionFunctions and with the product's adapter in its place."""
import json
import os
import subprocess

import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import CAM, GOLD, canon, crc, match_as_sets, oracle_for, poststep_frames, random_surfels


# the reference's SurfelMap is built into oracle/_ref/ only where the reference sources are; the pinned members below are
# also checked against CRC32s minted from it (tests/golden/reference_checksums.json), the other tests need it
needs_refmap = pytest.mark.skipif(not pyoracle.have_refmap(), reason="oracle/_ref/libdsm_refmap.so not built (needs the reference sources)")


def drive(m, n_frames, keyframe_every=1, seed0=1000, loops_at=None):
    """n frames of the synthetic drive through the node callbacks; every frame references the newest keyframe."""
    path, last_kf = [], 0
    for t in range(n_frames):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(CAM, seed0 + t, pose)
        p7 = pyoracle.pose_to_ros7(pose)
        is_kf = (t % keyframe_every) == 0
        m.frame(100.0 + 0.1 * t, gray, depth, p7, is_kf, last_kf if t else 0, path7=np.array(path).reshape(-1, 7),
                loops=loops_at(t) if loops_at else ())
        if is_kf or t == 0:
            path.append(p7)
            last_kf = m.num_poses() - 1


def golden_map(key):
    return json.load(open(os.path.join(GOLD, "reference_checksums.json")))["map"][key]


def warp_case():
    a = np.deg2rad(2.0)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    Wm[:3, 3] = [0.5, -0.1, 0.25]
    return random_surfels(5000, 3), np.ascontiguousarray(Wm.T.astype(np.float32).reshape(16))


def map_pins(m):
    """What the reference's SurfelMap `m` computes in the pinned cases below, as CRC32s (tests/golden/make_golden.py)."""
    pins = {"fuse_map_poststep": []}
    pool = np.zeros(0, SURFEL_DTYPE)
    for ref, gray, depth, pose in poststep_frames():
        m.set_local(pool)
        m.fuse_map(gray, depth, pose, ref)
        pool = m.local()
        pins["fuse_map_poststep"].append(crc(canon(pool)))
    pool, w = warp_case()
    m.set_local(pool)
    m.warp_active(w)
    pins["warp_active"] = crc(canon(m.local()))
    pins["mesh_vertices"] = crc(m.mesh_vertices(random_surfels(4000, 11)).tobytes())
    return pins


def test_fuse_map_poststep_is_pinned():
    """SurfelMap::fuse_map (surfel_map.cpp:1060-1113) == reference hot path + the restated post-step."""
    m = pyoracle.RefMap(CAM) if pyoracle.have_refmap() else None
    orc = oracle_for(CAM)
    pins = golden_map("fuse_map_poststep")
    pool = np.zeros(0, SURFEL_DTYPE)
    for t, (ref, gray, depth, pose) in enumerate(poststep_frames()):
        lo, no = orc.fuse(ref, gray, depth, pose, pool)
        want = pyoracle.fuse_map_poststep(lo, no)
        assert crc(canon(want)) == pins[t], f"frame {t}"
        if m is not None:
            m.set_local(pool)
            m.fuse_map(gray, depth, pose, ref)
            assert m.local().tobytes() == want.tobytes(), f"frame {t}"
        pool = want
    assert (lo["update_times"] == 0).sum() > 0
    if m is not None:
        m.close()


def test_warp_active_is_pinned():
    pool, w = warp_case()
    want = pyoracle.warp_active(pool, w)
    assert crc(canon(want)) == golden_map("warp_active")
    if pyoracle.have_refmap():
        m = pyoracle.RefMap(CAM)
        m.set_local(pool)
        m.warp_active(w)
        assert m.local().tobytes() == want.tobytes()
        m.close()


@needs_refmap
def test_move_add_surfels_and_cloud_builders_are_pinned(tmp_path):
    """A drive with a 1-pose drift-free window: keyframes leave the window, their surfels move to attached_surfels /
    inactive_pointcloud (surfel_map.cpp:1479-1497).  Checked member by member against the restatements."""
    m = pyoracle.RefMap(CAM, drift_free_poses=1)
    drive(m, 5)
    assert m.num_poses() == 5
    before = m.local()
    keep = set(m.local_pose_indexs())
    # 1. everything that left the window is attached to its pose, in pool order, and nowhere else
    n_att = 0
    for p in range(m.num_poses()):
        att = m.attached(p)
        n_att += len(att)
        if len(att):
            assert p not in keep and (att["last_update"] == p).all() and (att["update_times"] > 0).all()
    assert n_att > 0, "the drive never retired a keyframe"
    assert len(m.inactive_points()) == n_att
    assert not np.isin(before["last_update"][before["update_times"] > 0], [p for p in range(5) if p not in keep]).any()
    # 2. one more removal, by hand: shrink the window to the newest pose only and compare with the restated loop
    victim = sorted(keep)[0]
    m2_local, m2_out = pyoracle.retire(before, victim)
    if len(keep) > 1:
        # move_add_surfels(reference_index) recomputes the window around reference_index; with drift_free_poses=1 only
        # the reference pose and its direct neighbours stay -- use the newest pose as the root
        m.move_add_surfels(m.num_poses() - 1)
        after = m.local()
        gone = [p for p in keep if p not in set(m.local_pose_indexs())]
        want_local = before
        for p in gone:
            want_local, out = pyoracle.retire(want_local, p)
            assert m.attached(p).tobytes()[-len(out.tobytes()):] == out.tobytes() if len(out) else True
        assert after.tobytes() == want_local.tobytes()
    # 3. the cloud builders over the current state
    local = m.local()
    m.publish_clouds(m.num_poses() - 1)
    inactive = m.inactive_points()
    assert m.published("active_pointcloud").tobytes() == pyoracle.cloud_points(local, 5).tobytes()
    assert m.published("inactive_pointcloud").tobytes() == inactive.tobytes()
    assert m.published("pointcloud").tobytes() == np.concatenate([pyoracle.cloud_points(local, 5), inactive]).tobytes()
    nb = m.published("neighbor_pointcloud")
    live = pyoracle.cloud_points(local, 1)
    assert nb[:len(live)].tobytes() == live.tobytes()  # local part: update_times != 0 (:1291-1300)
    saved = m.save_cloud(str(tmp_path / "x.pcd"))
    assert saved.tobytes() == np.concatenate([pyoracle.cloud_points(local, 5), inactive]).tobytes()
    m.close()


@needs_refmap
def test_move_add_surfels_insertion_is_an_append():
    """A loop edge brings an old keyframe back into the drift-free window: its attached_surfels are appended to
    local_surfels in order and leave the inactive cloud (surfel_map.cpp:1526-1590) -- the semantics of
    dsm_pool_append / dsm_inactive_reactivate."""
    m = pyoracle.RefMap(CAM, drift_free_poses=2)
    drive(m, 5)
    att0, local_before, inactive_before = m.attached(0), m.local(), m.inactive_points()
    assert len(att0) > 0 and 0 not in m.local_pose_indexs()
    path = [pyoracle.pose_to_ros7(synth.pose_stream(t)) for t in range(5)]
    m.frame(100.5, None, None, pyoracle.pose_to_ros7(synth.pose_stream(5)), False, 4, path7=np.array(path), loops=[4, 0])
    window_before = m.local_pose_indexs()
    m.move_add_surfels(4)
    assert 0 in m.local_pose_indexs() and len(m.attached(0)) == 0
    # the same call retires whatever left the window rooted at pose 4 (removal runs before insertion)
    want_local, retired = local_before, []
    for p in [q for q in window_before if q not in m.local_pose_indexs()]:
        want_local, out = pyoracle.retire(want_local, p)
        assert m.attached(p).tobytes() == out.tobytes()
        retired.append(out)
    after = m.local()
    assert after.tobytes() == np.concatenate([want_local, att0]).tobytes()
    inactive_after = m.inactive_points()
    # pose 0 was the first segment of the inactive cloud: the rest moved down unchanged, new segments follow
    assert inactive_before[:len(att0)].tobytes() == pyoracle.cloud_points(att0, -(2 ** 31)).tobytes()
    want_inactive = np.concatenate([inactive_before[len(att0):]] + [pyoracle.cloud_points(o, -(2 ** 31)) for o in retired])
    assert inactive_after.tobytes() == want_inactive.tobytes()
    m.close()


def ros7_to_matrix(p7):
    from scipy.spatial.transform import Rotation
    T = np.eye(4)
    T[:3, :3] = Rotation.from_quat(p7[3:7]).as_matrix()
    T[:3, 3] = p7[:3]
    return T


@needs_refmap
def test_loop_closure_warps_the_active_surfels():
    """A corrected loop path arrives on the pose feed: orb_results_input -> warp_surfels (surfel_map.cpp:795-824) moves
    every active surfel by W = T_loop * T_cam^-1 of the oldest local keyframe.  Checks the restated warp (and the W
    the product's dsm_pool_transform is handed) against the node's own state, in the node's re-based world frame."""
    m = pyoracle.RefMap(CAM, drift_free_poses=10)
    drive(m, 4)
    before = m.local()
    path = [pyoracle.pose_to_ros7(synth.pose_stream(t)) for t in range(4)]
    a = np.deg2rad(1.5)
    C = np.eye(4)   # the correction the loop closure applies to every keyframe
    C[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    C[:3, 3] = [0.3, 0.0, -0.2]
    from scipy.spatial.transform import Rotation
    corrected = []
    for p7 in path:
        T = C @ ros7_to_matrix(p7)
        q = Rotation.from_matrix(T[:3, :3]).as_quat()
        corrected.append(np.concatenate([T[:3, 3], q]))
    pose4 = pyoracle.pose_to_ros7(synth.pose_stream(4))
    m.frame(100.4, None, None, pose4, True, 3, path7=np.array(corrected))   # pose feed only: no fuse after the warp
    after = m.local()
    assert len(after) == len(before)
    # the node re-bases the world with K = idea * T_first^-1 (surfel_map.cpp:214-232); in that frame W = K C K^-1
    idea = np.zeros((4, 4))
    idea[0, 0], idea[1, 2], idea[2, 1], idea[3, 3] = 1.0, 1.0, -1.0, 1.0
    K = idea @ np.linalg.inv(ros7_to_matrix(path[0]))
    Wm = K @ C @ np.linalg.inv(K)
    w = np.ascontiguousarray(Wm.T.astype(np.float32).reshape(16))
    want = pyoracle.warp_active(before, w)
    e = pyoracle.surfel_errors(after, want)
    assert e["pos"] < 2e-5 and e["nrm"] < 2e-5 and e["int_mismatch"] == 0, e
    moved = np.abs(after["px"] - before["px"]).max()
    assert moved > 0.05, "the loop correction did not move anything"
    m.close()


def test_product_mesh_writer_equals_reference_save_mesh(tmp_path):
    """dsm_write_ply_mesh / dsm_mesh_vertices (product, host code) against SurfelMap::save_mesh / push_a_surfel of the
    reference compiled in place: byte-identical file, bit-identical vertices.  The vertices are also pinned by the CRC32
    of the reference's; the file half needs the reference node itself."""
    s = random_surfels(4000, 11)
    v = capi.mesh_vertices(s)
    assert crc(v.tobytes()) == golden_map("mesh_vertices")
    assert pyoracle.mesh_vertices(s).tobytes() == v.tobytes()
    if not pyoracle.have_refmap():
        return
    m = pyoracle.RefMap(CAM, drift_free_poses=1)
    assert v.tobytes() == m.mesh_vertices(s).tobytes()
    drive(m, 5)
    ref_file, our_file = tmp_path / "ref.ply", tmp_path / "ours.ply"
    m.save_mesh(str(ref_file))
    local = m.local()
    surfels = np.concatenate([m.attached(p) for p in range(m.num_poses())] + [local[local["update_times"] >= 5]])
    assert len(surfels) > 100
    capi.write_ply_mesh(str(our_file), surfels)
    assert our_file.read_bytes() == ref_file.read_bytes()
    assert ref_file.read_text() == pyoracle.ply_mesh_text(surfels)
    m.close()


@needs_refmap
def test_three_line_patch_compiles_against_the_reference_source():
    """libdsm_refmap_b200.so is the reference's surfel_map.cpp, unmodified, with dsm::FusionFunctions in place of
    FusionFunctions (include path only): it exists, exports the driver, and takes the hot path from the C ABI."""
    if not pyoracle.have_refmap(b200=True):
        pytest.skip("libdsm_refmap_b200.so not built")
    path = os.path.join(pyoracle.REFDIR, "libdsm_refmap_b200.so")
    und = subprocess.run(["nm", "-D", "--undefined-only", path], capture_output=True, text=True).stdout
    assert " dsm_create" in und and " dsm_fuse_frame" in und
    dfn = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
    assert "dsmmap_frame" in dfn and "generate_super_pixels" not in dfn  # no CPU hot path inside


@needs_refmap
@pytest.mark.gpu
def test_reference_node_over_the_product_matches_the_reference_node():
    """The drop-in claim end to end: the same 6-frame drive through the reference's SurfelMap with its own CPU
    FusionFunctions and with the product library underneath.  Maps agree as sets within the surfel tolerance."""
    if not pyoracle.have_refmap(b200=True):
        pytest.skip("libdsm_refmap_b200.so not built")
    a, b = pyoracle.RefMap(CAM, drift_free_poses=2), pyoracle.RefMap(CAM, drift_free_poses=2, b200=True)
    drive(a, 6)
    drive(b, 6)
    assert a.num_poses() == b.num_poses() and a.local_pose_indexs() == b.local_pose_indexs()
    la, lb = a.local(), b.local()
    assert abs(len(la) - len(lb)) <= max(2, len(la) // 500)
    if len(la) == len(lb):
        match_as_sets(lb, la, tol=1e-3)
    for p in range(a.num_poses()):
        assert abs(len(a.attached(p)) - len(b.attached(p))) <= max(2, len(a.attached(p)) // 200)
    a.close()
    b.close()


@needs_refmap
@pytest.mark.gpu
def test_device_resident_map_tracks_the_reference_node():
    """System level, INTEGRATION.md steps 2+3: the reference node runs a drive on the CPU; the same frames go through
    the product with local_surfels AND attached_surfels resident on the device, replaying the node's own window
    decisions (which keyframes leave / re-enter).  After every frame the device's local pool and inactive store
    equal the node's local_surfels / inactive_pointcloud as sets, within the surfel tolerance."""
    ref = pyoracle.RefMap(CAM, drift_free_poses=2)
    ctx = capi.Context(CAM, max_batch=2, max_local_surfels=60000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.inactive_reserve(200000)
    idea = np.zeros((4, 4))
    idea[0, 0], idea[1, 2], idea[2, 1], idea[3, 3] = 1.0, 1.0, -1.0, 1.0
    K = idea @ np.linalg.inv(ros7_to_matrix(pyoracle.pose_to_ros7(synth.pose_stream(0))))  # surfel_map.cpp:214-232
    path, window_prev, stored = [], [], set()
    T = 7
    for t in range(T):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(CAM, 1000 + t, pose)
        p7 = pyoracle.pose_to_ros7(pose)
        ref_index = t - 1 if t else 0
        loops = [4, 0] if t == 5 else ()   # a loop edge 4-0 brings keyframe 0 back into the window at frame 5
        ref.frame(100.0 + 0.1 * t, gray, depth, p7, True, ref_index, path7=np.array(path).reshape(-1, 7), loops=loops)
        path.append(p7)
        window = ref.local_pose_indexs()
        for p in [q for q in window_prev if q not in window]:          # move_add_surfels: removal first ...
            if ctx.inactive_retire(p) > 0:
                stored.add(p)
        for p in [q for q in window if q not in window_prev and q in stored]:   # ... then insertion
            ctx.inactive_reactivate(p)
            stored.discard(p)
        window_prev = window
        fuse_pose = (K @ ros7_to_matrix(p7)).astype(np.float32)       # what synchronize_msgs hands to fuse_map
        ctx.fuse_frame_resident(ref_index, gray, depth, np.ascontiguousarray(fuse_pose.T.reshape(16)))
        want = ref.local()
        got = ctx.pool_download()
        got = got[got["update_times"] > 0]
        assert abs(len(got) - len(want)) <= max(2, len(want) // 300), f"frame {t}: {len(got)} vs {len(want)} local surfels"
        if len(got) == len(want):
            match_as_sets(got, want, tol=1e-3)
        n_in = ctx.inactive_size()[0]
        assert abs(n_in - len(ref.inactive_points())) <= max(2, n_in // 300), f"frame {t}: inactive {n_in}"
    assert ctx.inactive_size()[0] > 0, "the drive never retired a keyframe"
    ctx.close()
    ref.close()
