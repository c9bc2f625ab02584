"""dsm_fuse_stream_window: the node's per-frame move_add_surfels + fuse_map on the device, many frames per call.

Checked against (1) the per-call sequence dsm_inactive_retire / dsm_inactive_reactivate / dsm_fuse_frame_resident, byte
for byte after every call; (2) dsm_fuse_stream_resident when every list is empty; (3) the reference node itself over the
product (libdsm_refmap_window_b200.so), with the fuse poses and window lists the node used; plus the error contract."""
import functools
import os
import struct
import subprocess

import numpy as np
import pytest

import pyoracle
import pyoracle_window
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE

pytestmark = pytest.mark.gpu

CAM = synth.Camera(320, 240, 262.5, 262.5, 159.5, 119.5, 0.5, 30.0)
T = 16
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


def per_call(ctx, t0, t1, lists):
    """The existing calls, frame by frame: what dsm_fuse_stream_window must equal."""
    cnt = []
    for t in range(t0, t1):
        ref, rem, add = lists[t]
        for kf in rem:
            ctx.inactive_retire(kf)
        for kf in add:
            ctx.inactive_reactivate(kf)
        pose, gray, depth = frames()[t]
        cnt.append(ctx.fuse_frame_resident(ref, gray, depth, pose, want_count=True))
    return np.array(cnt, np.int32)


def windowed(ctx, t0, t1, lists, want_counts=True, empty=False):
    fr = frames()[t0:t1]
    ref = [lists[t][0] for t in range(t0, t1)]
    rem = [[] if empty else lists[t][1] for t in range(t0, t1)]
    add = [[] if empty else lists[t][2] for t in range(t0, t1)]
    return ctx.fuse_stream_window(ref, np.stack([f[1] for f in fr]), np.stack([f[2] for f in fr]),
                                  np.stack([capi.pose16(f[0]) for f in fr]), rem, add, want_counts=want_counts)


def state(ctx, kfs=range(T)):
    return (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes(), ctx.inactive_size(),
            ctx.inactive_export_cloud().tobytes(), ctx.inactive_export_poses(list(kfs)).tobytes())


def assert_same(a, b, what):
    for name, x, y in zip(("pool", "store", "size", "inactive cloud", "cloud by pose"), state(a), state(b)):
        assert x == y, f"{what}: {name} differs"


@needs_window_oracle
@pytest.mark.parametrize("chunk", [1, 3, 4, 8])
def test_window_stream_equals_per_call_sequence(chunk):
    lists = node_lists()
    assert any(len(r) >= 2 for _, r, _ in lists) and any(a for _, _, a in lists)
    a, b = new_ctx(), new_ctx()
    for t0 in range(0, T, chunk):
        t1 = min(T, t0 + chunk)
        want = per_call(a, t0, t1, lists)
        got = windowed(b, t0, t1, lists)
        assert got.tolist() == want.tolist(), f"frames {t0}-{t1}: new surfels per frame"
        assert_same(a, b, f"after frames {t0}-{t1}")
    assert a.inactive_size()[0] > 0
    a.close()
    b.close()


@needs_window_oracle
@pytest.mark.parametrize("max_batch,chunk", [(8, 4), (16, 8)])
def test_alternating_halves_without_synchronisation(max_batch, chunk):
    """Calls without counts never wait for the device; with 2 * chunk <= max_batch consecutive calls use alternate
    staging halves, so the window tables of one call are staged while the previous call's frames still run."""
    lists = node_lists()
    a, b = new_ctx(), new_ctx(max_batch=max_batch)
    per_call(a, 0, T, lists)
    for t0 in range(0, T, chunk):
        windowed(b, t0, t0 + chunk, lists, want_counts=False)
    assert_same(a, b, "end of the drive")
    a.close()
    b.close()


@needs_window_oracle
def test_empty_lists_equal_fuse_stream_resident():
    lists = node_lists()
    a, b = new_ctx(), new_ctx()
    for t0 in range(0, T, 4):
        fr = frames()[t0:t0 + 4]
        want = a.fuse_stream_resident([lists[t][0] for t in range(t0, t0 + 4)], np.stack([f[1] for f in fr]),
                                      np.stack([f[2] for f in fr]), np.stack([capi.pose16(f[0]) for f in fr]), want_counts=True)
        got = windowed(b, t0, t0 + 4, lists, empty=True)
        assert got.tolist() == want.tolist()
        assert a.pool_download().tobytes() == b.pool_download().tobytes()
    a.close()
    b.close()


@needs_window_oracle
def test_inactive_calls_after_windowed_calls():
    """The existing dsm_inactive_* calls see the store a windowed call left, including an asynchronous
    dsm_inactive_transform issued straight after it (its keyframe's range is found on the device)."""
    lists = node_lists()
    a, b = new_ctx(), new_ctx()
    per_call(a, 0, 12, lists)
    windowed(b, 0, 8, lists, want_counts=False)
    windowed(b, 8, 12, lists, want_counts=False)
    ang = np.deg2rad(1.5)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]]
    Wm[:3, 3] = [0.1, -0.2, 0.05]
    stored = sorted({kf for _, r, _ in lists[:12] for kf in r})
    for kf in stored:
        a.inactive_transform(kf, Wm)
        b.inactive_transform(kf, Wm)   # b: straight after the windowed call, nothing synchronised yet
    assert_same(a, b, "after the inactive warp")
    kf = next(k for k in stored if len(a.inactive_download(k)))
    assert a.inactive_reactivate(kf) == b.inactive_reactivate(kf) > 0
    assert a.inactive_retire(kf) == b.inactive_retire(kf)
    assert_same(a, b, "after a reactivation and a retirement")
    # and the windowed call continues from the state the per-call calls left
    per_call(a, 12, T, lists)
    windowed(b, 12, T, lists)
    assert_same(a, b, "end of the drive")
    a.close()
    b.close()


def test_invalid_lists_and_state_errors():
    ctx = new_ctx(store=0)
    pose, gray, depth = frames()[0]
    g, d, p = gray[None], depth[None], capi.pose16(pose)[None]

    def call(rem, add, c=ctx, n=1):
        with pytest.raises(capi.DsmError) as e:
            c.fuse_stream_window([0] * n, np.repeat(g, n, 0), np.repeat(d, n, 0), np.repeat(p, n, 0), rem, add)
        return e.value.code

    assert call([[1]], [[]]) == -7                                    # non-empty list, no store reserved
    ctx.inactive_reserve(1000)
    assert call([[-1]], [[]]) == -1                                   # negative keyframe
    assert call([[2, 2]], [[]]) == -1                                 # twice in one list
    assert call([[3]], [[3]]) == -1                                   # in both lists
    assert call([list(range(capi.WINDOW_MAX_KEYS + 1))], [[]]) == -1  # too many keys
    keys, ofs = np.array([1, 2], np.int32), np.array([0, 2, 1], np.int32)  # offsets going down
    rc = ctx.lib.dsm_fuse_stream_window(ctx.h, 2, capi._ptr(np.zeros(2, np.int32)), capi._ptr(np.repeat(g, 2, 0)),
                                        capi._ptr(np.repeat(d, 2, 0)), capi._ptr(np.repeat(p, 2, 0)), capi._ptr(keys),
                                        capi._ptr(ofs), None, None, None)
    assert rc == -1
    assert ctx.pool_size() == 0  # nothing was enqueued
    ctx.close()


@needs_window_oracle
def test_pool_overflow_stops_at_the_last_frame_that_fits():
    """A capacity one surfel short of frame 5's worst case: frames 0-4 are applied, 5-7 are not (n_new = -1), and the
    pool and store are those after frame 4.  The word stays set until a call reads it."""
    from densesurfelmapping_b200.elements import num_seeds
    lists = node_lists()
    a = new_ctx()
    counts = per_call(a, 0, 5, lists)
    cap = a.pool_size() + num_seeds(CAM.width, CAM.height) - 1
    b = new_ctx(cap=cap)
    with pytest.raises(capi.DsmError) as e:
        windowed(b, 0, 8, lists)
    assert e.value.code == -6
    got = e.value.counts
    assert got[:5].tolist() == counts.tolist() and (got[5:] == -1).all(), got
    assert_same(a, b, "after the rejected frame")
    # without counts the call returns at once; the next read reports the rejection and clears it
    windowed(b, 5, 6, lists, want_counts=False)
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6
    assert_same(a, b, "after the second rejection")
    a.close()
    b.close()


@needs_window_oracle
def test_store_overflow_is_reported_by_the_next_read_and_resumes():
    lists = node_lists()
    first = next(t for t in range(T) if lists[t][1])  # first frame that retires
    a = new_ctx()
    per_call(a, 0, first, lists)
    b = new_ctx(store=1)                               # any retirement of a live surfel overflows
    windowed(b, 0, first + 2, lists, want_counts=False)
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6
    assert_same(a, b, "after the rejected frame")
    # resume: the next frames with empty lists, on both
    fr = frames()[first:first + 2]
    a.fuse_stream_resident([lists[t][0] for t in (first, first + 1)], np.stack([f[1] for f in fr]), np.stack([f[2] for f in fr]),
                           np.stack([capi.pose16(f[0]) for f in fr]))
    got = windowed(b, first, first + 2, lists, empty=True)
    assert (got >= 0).all()
    assert_same(a, b, "after the resumed frames")
    a.close()
    b.close()


def ros7_to_matrix(p7):
    x, y, z, qx, qy, qz, qw = p7
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw)],
                  [2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw)],
                  [2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)]])
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = R, [x, y, z]
    return M


@pytest.mark.skipif(not pyoracle_window.have_refmap_window(b200=True), reason="libdsm_refmap_window_b200.so not built")
@pytest.mark.parametrize("chunk", [1, 4, "per_call"])
def test_product_equals_the_reference_node(chunk):
    """The reference node over the product (its own move_add_surfels and host post-step, the product's fuse kernels)
    against dsm_fuse_stream_window fed with the fuse poses and window lists that node used: local_surfels slot for slot,
    attached_surfels and inactive_pointcloud byte for byte.  "per_call": the same frames through dsm_inactive_retire /
    dsm_inactive_reactivate / dsm_fuse_frame_resident, one call each."""
    m = pyoracle_window.RefMapWindow(CAM, drift_free_poses=2, b200=True)
    path, last_kf, rec = [], 0, []
    for t in range(T):
        is_kf, ref, loops = schedule(t)
        pose, gray, depth = frames()[t]
        p7 = pyoracle.pose_to_ros7(pose)
        root = (last_kf if t else 0) if ref == "new" else ref
        m.frame(100.0 + 0.1 * t, None, None, p7, is_kf or t == 0, root, path7=np.array(path).reshape(-1, 7), loops=loops)
        if is_kf or t == 0:
            path.append(p7)
            last_kf = m.num_poses() - 1
        pending = m.pending_frame()
        assert pending is not None and pending[0] == root
        m.images(100.0 + 0.1 * t, gray, depth)
        rec.append(pending)
    assert any(r for _, _, r, _ in rec) and any(a for _, _, _, a in rec)
    ctx = new_ctx()
    if chunk == "per_call":
        for (ref, pose, rem, add), (_, gray, depth) in zip(rec, frames()):
            for kf in rem:
                ctx.inactive_retire(kf)
            for kf in add:
                ctx.inactive_reactivate(kf)
            ctx.fuse_frame_resident(ref, gray, depth, pose)
    else:
        for t0 in range(0, T, chunk):
            part = rec[t0:t0 + chunk]
            fr = frames()[t0:t0 + chunk]
            ctx.fuse_stream_window([r[0] for r in part], np.stack([f[1] for f in fr]), np.stack([f[2] for f in fr]),
                                   np.stack([r[1] for r in part]), [r[2] for r in part], [r[3] for r in part])
    assert ctx.pool_download().tobytes() == m.local().tobytes()
    for p in range(m.num_poses()):
        assert ctx.inactive_download(p).tobytes() == m.attached(p).tobytes(), f"attached_surfels of pose {p}"
    pts = ctx.inactive_export_cloud()
    assert pts.view(np.float32).reshape(-1, 4).tobytes() == m.inactive_points().tobytes()
    assert len(pts) > 0
    ctx.close()
    m.close()


@needs_window_oracle
def test_cpp_caller_of_the_windowed_fuse_map(tmp_path):
    """tests/cpp/window_main.cpp: dsm::ResidentSurfelPool::fuse_map with the two lists, one frame per call, never
    synchronising; the map it reads back at the end equals the Python binding's chunk-of-1 run."""
    from test_cpp_adapter import build_adapter
    exe = build_adapter("window_main")
    lists = node_lists()
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<i", T))
        for t in range(T):
            ref, rem, add = lists[t]
            pose, gray, depth = frames()[t]
            f.write(struct.pack("<i", ref) + capi.pose16(pose).tobytes())
            f.write(struct.pack("<i", len(rem)) + np.asarray(rem, np.int32).tobytes())
            f.write(struct.pack("<i", len(add)) + np.asarray(add, np.int32).tobytes())
            f.write(gray.tobytes() + depth.tobytes())
    args = [exe, str(CAM.width), str(CAM.height)] + [repr(float(v)) for v in (CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.far, CAM.near)]
    r = subprocess.run(args + [fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw, arrs, o = open(fout, "rb").read(), [], 0
    for dt in (SURFEL_DTYPE, SURFEL_DTYPE, POINT_DTYPE):
        n = struct.unpack_from("<i", raw, o)[0]
        arrs.append(np.frombuffer(raw, dt, n, o + 4))
        o += 4 + n * dt.itemsize
    ctx = new_ctx(max_batch=2, cap=400000, store=400000)
    for t in range(T):
        windowed(ctx, t, t + 1, lists, want_counts=False)
    assert arrs[0].tobytes() == ctx.pool_download().tobytes()
    assert arrs[1].tobytes() == ctx.inactive_download(-1).tobytes()
    assert arrs[2].tobytes() == ctx.inactive_export_cloud().tobytes()
    assert len(arrs[1]) > 0
    ctx.close()
    assert os.path.exists(exe)
