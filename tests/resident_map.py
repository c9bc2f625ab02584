"""The GPU-resident map the GPU tests drive: the drive's camera and frames, the node's window lists, a context with its
pool and store, windowed calls, loop-closure warps, the readers that tests compare byte for byte, and the checks of
published clouds and distance fields against their oracles."""
import functools

import numpy as np
import pytest

import pyoracle
import pyoracle_publish
import pyoracle_window
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import CAM

T = 16
STORE = 1 << 18
needs_window_oracle = pytest.mark.skipif(not pyoracle_window.have_refmap_window(),
                                         reason="oracle/_ref/libdsm_refmap_window.so not built (needs the reference sources)")


def schedule(t):
    """(is_keyframe, reference, loops) of frame t: a keyframe every other frame, a loop edge 4 <-> 0 at frame 9, the
    reference jumping back to keyframe 1 at frames 12-13 (several keyframes leave at once, old ones return)."""
    return t % 2 == 0, (1 if t in (12, 13) else "new"), ([4, 0] if t == 9 else [])


@functools.lru_cache(maxsize=None)
def frames():
    out = []
    for t in range(T):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(CAM, 2000 + t, pose)
        out.append((pose, gray, depth))
    return out


@functools.lru_cache(maxsize=None)
def node_lists(drift_free_poses=2):
    """(reference index, poses_to_remove, poses_to_add) per frame, from the reference node's own get_add_remove_poses
    and move_add_surfels on the pose graph of the drive."""
    m = pyoracle_window.RefMapWindow(CAM, drift_free_poses=drift_free_poses)
    path, last_kf, out = [], 0, []
    for t in range(T):
        is_kf, ref, loops = schedule(t)
        p7 = pyoracle.pose_to_ros7(synth.pose_stream(t))
        root = (last_kf if t else 0) if ref == "new" else ref
        m.frame(100.0 + 0.1 * t, None, None, p7, is_kf or t == 0, root, path7=np.array(path).reshape(-1, 7), loops=loops)
        if is_kf or t == 0:
            path.append(p7)
            last_kf = m.num_poses() - 1
        rem, add = m.window_lists(root)
        m.move_add_surfels(root)
        out.append((root, rem, add))
    m.close()
    return tuple(out)


def new_ctx(max_batch=16, cap=1 << 18, store=1 << 18):
    ctx = capi.Context(CAM, max_batch=max_batch, max_local_surfels=cap)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    if store:
        ctx.inactive_reserve(store)
    return ctx


def windowed(ctx, t0, t1, lists, want_counts=True, empty=False):
    fr = frames()[t0:t1]
    ref = [lists[t][0] for t in range(t0, t1)]
    rem = [[] if empty else lists[t][1] for t in range(t0, t1)]
    add = [[] if empty else lists[t][2] for t in range(t0, t1)]
    return ctx.fuse_stream_window(ref, np.stack([f[1] for f in fr]), np.stack([f[2] for f in fr]),
                                  np.stack([capi.pose16(f[0]) for f in fr]), rem, add, want_counts=want_counts)


def warp(k=1):
    ang = np.deg2rad(1.5 * k)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]]
    Wm[:3, 3] = [0.1 * k, -0.2, 0.05]
    return Wm


def simple_lists():
    """(reference, retire, reactivate) per frame without the reference node: a keyframe every other frame, a window of
    two keyframes; keyframe 0 comes back at frame 9, leaves at 11, comes back with keyframe 1 at 13, and frame 14
    retires three keyframes at once."""
    out = []
    for t in range(T):
        ref = t // 2
        rem = [ref - 2] if t % 2 == 0 and ref >= 2 else []
        add = []
        if t == 9:
            add = [0]
        if t == 11:
            rem = [0]
        if t == 13:
            add = [0, 1]
        if t == 14:
            rem = [5, 0, 1]
        out.append((ref, rem, add))
    return tuple(out)


class Mirror:
    """The host's view across snapshots: the model's shadow and the previous size."""

    def __init__(self, cap=STORE):
        self.shadow, self.prev = np.zeros((cap, 4), np.float32), 0

    def check(self, ctx, inactive, changed_from, what):
        pts = inactive.view(np.float32).reshape(-1, 4)
        chunks, want, self.shadow = pyoracle_publish.mirror_step(self.shadow, self.prev, pts)
        assert changed_from == want, f"{what}: inactive_changed_from {changed_from}, the clouds first differ at {want}"
        assert ctx.publish_chunks() == len(chunks), f"{what}: forwarded chunks"
        self.prev = len(pts)
        return chunks


def snapshot_equals_readers(ctx, mirror, what, min_update_times=5):
    ctx.publish_enqueue(min_update_times)
    active, inactive, cf = ctx.publish_wait()
    assert active.tobytes() == ctx.pool_export_cloud(min_update_times).tobytes(), f"{what}: active cloud"
    assert inactive.tobytes() == ctx.inactive_export_cloud().tobytes(), f"{what}: inactive cloud"
    mirror.check(ctx, inactive, cf, what)
    return active, inactive, cf


# ---- checkpoints ----
CONSTANTS = {"drive": capi.CONSTANTS_DRIVE, "rgbd": capi.CONSTANTS_RGBD}
# save point k (frames 0..k-1 fused) of simple_lists(), and a loop-closure warp issued right before the save or right
# after the load
SAVES = {"after_retirement": (5, None), "after_reactivation": (14, None), "keyframe0_back": (10, None),
         "after_transforms": (8, "before"), "warp_after_load": (12, "after")}


def readers(ctx):
    return (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes(), ctx.inactive_segments().tobytes(),
            ctx.inactive_export_cloud().tobytes(), ctx.pool_export_cloud(5).tobytes())


def run(ctx, lists, t0, t1, chunk):
    for s in range(t0, t1, chunk):
        windowed(ctx, s, min(t1, s + chunk), lists, want_counts=False)


def loop_warp(ctx, kfs):
    ctx.pool_transform(warp(1))
    for kf in kfs:
        ctx.inactive_transform(kf, warp(2))


def stored_keyframes(ctx):
    return sorted(set(ctx.inactive_segments()[:, 0].tolist()))


def made(constants="drive", **kw):
    ctx = new_ctx(**kw)
    ctx.set_constants(CONSTANTS[constants])
    return ctx


# ---- distance fields ----
SHAPES = [(37, 41, 13), (64, 64, 32), (1, 1, 1), (128, 1, 7)]
COMBOS = [(m, v) for m in (1, 5) for v in (0.125, 0.1, 0.3)]


def xyz(*clouds):
    return np.concatenate([c.view(np.float32).reshape(-1, 4)[:, :3] for c in clouds])


def camera(t):
    return frames()[t][0][12:15].astype(np.float64)


def field_points(ctx, m):
    return xyz(ctx.pool_export_cloud(m), ctx.inactive_export_cloud())


def assert_field(got, want, what):
    dist, origin, n_occ = got
    assert origin.tolist() == want[1].tolist(), f"{what}: origin"
    assert n_occ == want[2], f"{what}: occupied voxels {n_occ}, want {want[2]}"
    assert dist.shape == want[0].shape and dist.tobytes() == want[0].tobytes(), \
        f"{what}: {(dist.view(np.uint32) != want[0].view(np.uint32)).sum()} voxels differ"


def centres(ctx, t, voxel, shape, m):
    """At the camera of frame t; on the edge of the map's bounding box, so that half of the grid lies beyond it; far
    outside it, so that nothing is occupied; and in the middle of the voxel of an obstacle point, so that even a grid of
    one voxel is occupied."""
    pts = field_points(ctx, 1)
    lo, hi = pts.min(0).astype(np.float64), pts.max(0).astype(np.float64)
    edge = (lo + hi) / 2
    edge[0] = hi[0]
    far = hi + np.array(shape) * voxel + 100.0
    obstacles = field_points(ctx, m)   # none before the first surfel reaches m updates
    cell = None
    if len(obstacles):
        cell = (np.floor(obstacles[len(obstacles) // 2] / np.float32(voxel)).astype(np.float64) + 0.5) * float(np.float32(voxel))
    return [("camera", camera(t)), ("half off the map", edge), ("off the map", far), ("on an obstacle", cell)]


def map_state(ctx):
    return (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes(), ctx.inactive_segments().tobytes())
