"""The node's per-frame window step (SurfelMap::move_add_surfels, surfel_map.cpp:1458-1595), restated in numpy on the
pool, the inactive store and its segment list (oracle/pyoracle_window.WindowModel) -- the semantics
dsm_fuse_stream_window implements on the device -- pinned byte for byte against the reference node's own
move_add_surfels (libdsm_refmap_window.so: local_surfels, every pose's attached_surfels, inactive_pointcloud)."""
import numpy as np
import pytest

import pyoracle
import pyoracle_window
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE

CAM = synth.Camera(320, 240, 262.5, 262.5, 159.5, 119.5, 0.5, 30.0)

needs_window_oracle = pytest.mark.skipif(not pyoracle_window.have_refmap_window(),
                                         reason="oracle/_ref/libdsm_refmap_window.so not built (needs the reference sources)")


def schedule(n_frames=22):
    """(is_keyframe, reference, loops) per frame.  reference: 'new' = the newest keyframe, or a keyframe index.
    A keyframe every other frame along a chain; frame 9 closes a loop to keyframe 0; frames 12-13 are referenced to
    keyframe 1 (the window jumps back: several keyframes leave at once, old ones return), then the drive moves on
    (the returned ones leave again)."""
    out = []
    for t in range(n_frames):
        ref = 1 if t in (12, 13) else "new"
        out.append((t % 2 == 0, ref, [4, 0] if t == 9 else []))
    return out


def surfels_for(rng, kf, n, t):
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
        s[f] = rng.standard_normal(n).astype(np.float32)
    s["px"] += np.float32(t)
    s["update_times"] = rng.integers(1, 9, n)
    s["last_update"] = kf
    return s


def drive_window(m, drift_free_poses, seed=7, no_surfels_kf=6, check=None):
    """Pose feeds through the node's callback, synthetic fuse results in between (new surfels carrying the reference
    index, some surfels dying), and each frame's window step on the reference node and on the model."""
    rng = np.random.default_rng(seed)
    model = pyoracle_window.WindowModel()
    path, last_kf, seen = [], 0, []
    for t, (is_kf, ref, loops) in enumerate(schedule()):
        pose = synth.pose_stream(t)
        p7 = pyoracle.pose_to_ros7(pose)
        root = (last_kf if t else 0) if ref == "new" else ref
        m.frame(100.0 + 0.1 * t, None, None, p7, is_kf or t == 0, root, path7=np.array(path).reshape(-1, 7), loops=loops)
        if is_kf or t == 0:
            path.append(p7)
            last_kf = m.num_poses() - 1
        # what the previous fuse left: new surfels of this frame's reference keyframe, a few deaths
        pool = model.pool.copy()
        if len(pool):
            pool["update_times"][rng.random(len(pool)) < 0.05] = 0
        if root != no_surfels_kf:
            pool = np.concatenate([pool, surfels_for(rng, root, int(rng.integers(20, 60)), t)])
        model.pool = pool
        m.set_local(pool)
        retire, react = m.window_lists(root)
        live = model.pool["last_update"][model.pool["update_times"] > 0]
        empty = [kf for kf in retire if not (live == kf).any()]  # retired without a single surfel
        m.move_add_surfels(root)
        model.step(retire, react)
        seen.append((retire, react, empty))
        assert m.local().tobytes() == model.pool.tobytes(), f"frame {t}: local_surfels"
        for p in range(m.num_poses()):
            assert m.attached(p).tobytes() == model.attached(p).tobytes(), f"frame {t}: attached_surfels of pose {p}"
        assert m.inactive_points().tobytes() == pyoracle_window.cloud(model.store).tobytes(), f"frame {t}: inactive_pointcloud"
        if check:
            check(t, model)
    return seen, model


@needs_window_oracle
@pytest.mark.parametrize("drift_free_poses", [1, 2, 3])
def test_window_model_is_pinned_to_move_add_surfels(drift_free_poses):
    m = pyoracle_window.RefMapWindow(CAM, drift_free_poses=drift_free_poses)
    seen, model = drive_window(m, drift_free_poses)
    m.close()
    retired = [kf for r, _, _ in seen for kf in r]
    returned = [kf for _, a, _ in seen for kf in a]
    assert len(seen) >= 12
    assert any(len(r) >= 2 for r, _, _ in seen), "no frame retires several keyframes"
    assert returned, "no keyframe re-entered the window"
    assert any(retired.count(k) >= 2 and k in returned for k in set(retired)), "no keyframe retired, reactivated, retired again"
    assert any(e for _, _, e in seen), "no keyframe without surfels was retired"


@needs_window_oracle
def test_loop_edge_brings_an_old_keyframe_back():
    """Frame 9's loop edge (keyframe 4 <-> 0) puts keyframe 0 back into a 2-pose window rooted at keyframe 4."""
    m = pyoracle_window.RefMapWindow(CAM, drift_free_poses=2)
    seen, _ = drive_window(m, 2)
    m.close()
    assert 0 in seen[9][1]


def test_window_lists_pack_into_offsets():
    keys, ofs = capi.window_lists([[3, 1], [], [7]])
    assert ofs.tolist() == [0, 2, 2, 3] and keys[:3].tolist() == [3, 1, 7]


def test_window_model_keeps_store_order():
    """Hand-made case: two retirements, then one reactivation from the middle of the store."""
    pool = np.zeros(6, SURFEL_DTYPE)
    pool["update_times"] = [1, 2, 0, 3, 4, 5]
    pool["last_update"] = [1, 2, 1, 1, 3, 2]
    pool["px"] = np.arange(6)
    m = pyoracle_window.WindowModel(pool)
    m.step([2, 1], [])
    assert m.segs == [(2, 0, 2), (1, 2, 2)]
    assert m.store["px"].tolist() == [1, 5, 0, 3]
    assert m.pool["update_times"].tolist() == [0, 0, 0, 0, 4, 0]
    m.step([3], [2])
    assert m.segs == [(1, 0, 2), (3, 2, 1)]
    assert m.store["px"].tolist() == [0, 3, 4]
    assert m.pool["px"].tolist() == [0, 1, 2, 3, 4, 5, 1, 5]
