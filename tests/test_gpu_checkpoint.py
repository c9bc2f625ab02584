"""Checkpoint and resume of the GPU-resident map (dsm_map_save / dsm_map_load, dsm_inactive_segments / _load).

A drive resumed from a checkpoint is byte-identical to the same drive run without interruption: pool, store, segment
table and both clouds after every call; the file holds exactly what the readers return; every refused load leaves the map
as it was; the first snapshot after a load forwards the whole inactive cloud; and dsm::SurfelMapNode resumes from its
own checkpoint (tests/cpp/checkpoint_main.cpp)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from test_checkpoint_format import parse
from test_gpu_publish import Mirror, simple_lists, snapshot_equals_readers, warp
from test_gpu_window_stream import CAM, T, new_ctx, windowed
from test_surfel_node import Script, drive

pytestmark = pytest.mark.gpu

STORE = 1 << 18
CONSTANTS = {"drive": capi.CONSTANTS_DRIVE, "rgbd": capi.CONSTANTS_RGBD}
# save point k (frames 0..k-1 fused) of simple_lists(), and a loop-closure warp issued right before the save or right
# after the load
SAVES = {"after_retirement": (5, None), "after_reactivation": (14, None), "keyframe0_back": (10, None),
         "after_transforms": (8, "before"), "warp_after_load": (12, "after")}


def readers(ctx):
    return (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes(), ctx.inactive_segments().tobytes(),
            ctx.inactive_export_cloud().tobytes(), ctx.pool_export_cloud(5).tobytes())


def assert_same(a, b, what):
    for name, x, y in zip(("pool", "store", "segments", "inactive cloud", "active cloud"), readers(a), readers(b)):
        assert x == y, f"{what}: {name} differs"


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


@pytest.mark.parametrize("save", sorted(SAVES))
@pytest.mark.parametrize("chunk", [1, 4, 8])
@pytest.mark.parametrize("constants", ["drive", "rgbd"])
def test_resume_equals_the_uninterrupted_drive(tmp_path, save, chunk, constants):
    lists = simple_lists()
    k, when = SAVES[save]
    if save == "after_retirement":
        assert lists[k - 1][1] and not lists[k - 1][2]
    if save == "after_reactivation":
        assert len(lists[k - 1][2]) >= 2
    if save == "keyframe0_back":
        assert lists[k - 1][2] == [0]
    a = made(constants, store=STORE)
    run(a, lists, 0, k, chunk)
    if when == "before":
        loop_warp(a, stored_keyframes(a))
    path = str(tmp_path / "map.dsm")
    a.map_save(path, extra=b"resume")
    b = made(constants, store=STORE)
    assert b.map_load(path) == b"resume"
    assert_same(a, b, "right after the load")
    assert len(a.inactive_segments()) > 0
    if when == "after":
        kfs = stored_keyframes(a)
        loop_warp(a, kfs)
        loop_warp(b, kfs)
    for s in range(k, T, chunk):
        for c in (a, b):
            windowed(c, s, min(T, s + chunk), lists, want_counts=False)
        assert_same(a, b, f"frames {s}-{min(T, s + chunk) - 1} after the load at {k}")
    a.close()
    b.close()


def test_the_file_is_the_readers(tmp_path):
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    run(ctx, lists, 0, 11, 4)
    path = tmp_path / "map.dsm"
    ctx.map_save(str(path), extra=b"\x01\x02\x03")
    h, pool, store, table, extra, ok = parse(path.read_bytes())
    assert ok, "checksum"
    assert pool.tobytes() == ctx.pool_download().tobytes()
    assert store.tobytes() == ctx.inactive_download(-1).tobytes()
    assert table.tobytes() == ctx.inactive_segments().tobytes()
    assert table[:, 2].sum() == len(store) > 0 and extra == b"\x01\x02\x03"
    assert (h["width"], h["height"]) == (CAM.width, CAM.height)
    assert tuple(h["constants"]) == capi.CONSTANTS_DRIVE
    assert [n for n in os.listdir(tmp_path)] == ["map.dsm"]       # no temporary left behind
    # without a store: an empty store section
    bare = new_ctx(store=0)
    run(bare, lists, 0, 3, 3)
    bare.map_save(str(tmp_path / "bare.dsm"))
    h, pool, store, table, extra, ok = parse((tmp_path / "bare.dsm").read_bytes())
    assert ok and len(store) == len(table) == len(extra) == 0 and pool.tobytes() == bare.pool_download().tobytes()
    ctx.close()
    bare.close()


def full_state(ctx):
    st = [ctx.pool_download().tobytes(), ctx.pool_export_cloud(5).tobytes()]
    try:
        st += [ctx.inactive_download(-1).tobytes(), ctx.inactive_segments().tobytes(), ctx.inactive_export_cloud().tobytes()]
    except capi.DsmError as e:   # no store: DSM_E_STATE
        st.append(e.code)
    return st


def load_code(ctx, path, cap=1 << 10):
    buf, n = ctypes.create_string_buffer(cap), ctypes.c_size_t(0)
    return ctx.lib.dsm_map_load(ctx.h, os.fsencode(path), buf, cap, ctypes.byref(n)), n.value


def test_refused_loads_leave_the_map_as_it_was(tmp_path):
    lists = simple_lists()
    src = new_ctx(store=STORE)
    run(src, lists, 0, 10, 4)
    n_pool, (n_store, _) = src.pool_size(), src.inactive_size()
    path = str(tmp_path / "map.dsm")
    src.map_save(path, extra=b"x" * 40)
    raw = open(path, "rb").read()

    def refused(ctx, p, code, cap=1 << 10):
        before = full_state(ctx)
        rc, _ = load_code(ctx, p, cap)
        assert rc == code, (p, rc, code)
        assert full_state(ctx) == before, f"load of {p} changed the map"

    def target(cam=CAM, cap=1 << 18, store=STORE, own=True):
        c = capi.Context(cam, max_batch=16, max_local_surfels=cap)
        c.pool_upload(np.zeros(0, SURFEL_DTYPE))
        if store:
            c.inactive_reserve(store)
        if own:
            run(c, lists, 0, 6, 3)     # a map of its own, which a refused load must keep
        return c

    other = synth.Camera(CAM.width, CAM.height, CAM.fx + 1, CAM.fy, CAM.cx, CAM.cy, CAM.near, CAM.far)
    c = target(other)
    refused(c, path, -1)                                  # geometry
    c.close()
    c = target()
    c.set_constants(capi.CONSTANTS_RGBD)
    refused(c, path, -1)                                  # constants
    c.close()
    c = target(cap=n_pool - 1, own=False)
    c.pool_upload(src.pool_download()[:n_pool // 2])
    refused(c, path, -6)                                  # pool over max_local_surfels
    c.close()
    c = target(store=n_store - 1, own=False)
    refused(c, path, -6)                                  # store over the reservation
    c.close()
    c = target(store=0, own=False)
    c.pool_upload(src.pool_download()[:100])
    refused(c, path, -7)                                  # stored surfels, no store
    c.close()
    c = target()
    for name, data, code in [("truncated", raw[:-100], -9), ("short", raw[:50], -9),
                             ("flipped", raw[:200] + bytes([raw[200] ^ 4]) + raw[201:], -9),
                             ("magic", b"Y" + raw[1:], -1)]:
        p = str(tmp_path / f"{name}.dsm")
        with open(p, "wb") as f:
            f.write(data)
        refused(c, p, code)
    refused(c, str(tmp_path / "missing.dsm"), -9)
    before = full_state(c)
    rc, n = load_code(c, path, cap=39)                    # extra_cap one byte short: the size comes back
    assert rc == -6 and n == 40 and full_state(c) == before
    c.publish_enable()
    c.publish_enqueue(5)
    refused(c, path, -7)                                  # a snapshot in flight
    c.publish_wait()
    assert c.map_load(path) == b"x" * 40
    assert_same(src, c, "after the load that was finally accepted")
    c.close()
    src.close()


def test_inactive_load_checks_its_table():
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    run(ctx, lists, 0, 10, 4)
    store, table = ctx.inactive_download(-1), ctx.inactive_segments()
    assert len(table) >= 2
    L = ctx.lib

    def code(s, t, c=ctx):
        s = np.ascontiguousarray(s, SURFEL_DTYPE)
        t = np.ascontiguousarray(t, np.int32).reshape(-1, 3)
        return L.dsm_inactive_load(c.h, capi._ptr(s) if len(s) else None, len(s), capi._ptr(t) if len(t) else None, len(t))

    before = full_state(ctx)
    bad = []
    t = table.copy(); t[0, 1] = 1; bad.append(t)                          # not from 0
    t = table.copy(); t[1, 1] += 1; bad.append(t)                         # not contiguous
    t = table.copy(); t[-1, 2] -= 1; bad.append(t)                        # counts short of n
    t = table.copy(); t[0, 0] = -1; bad.append(t)                         # negative keyframe
    t = np.vstack([table, [[table[0, 0], len(store), 0]]]); bad.append(t)  # a count of 0
    for t in bad:
        assert code(store, t) == -1, t
    s = store.copy(); s["update_times"][0] = 0
    assert code(s, table) == -1                                           # a dead stored surfel
    s = store.copy(); s["last_update"][-1] += 1
    assert code(s, table) == -1                                           # last_update of another keyframe
    big = new_ctx(store=len(store) - 1)
    assert code(store, table, big) == -6                                  # over the reservation
    none = new_ctx(store=0)
    assert code(store, table, none) == -7                                 # no reservation
    ctx.publish_enable()
    ctx.publish_enqueue(5)
    assert code(store, table) == -7                                       # a snapshot in flight
    ctx.publish_wait()
    assert full_state(ctx) == before
    # a keyframe owning two segments is accepted, and an empty load empties the store
    kf = int(table[0, 0])
    s = store.copy(); s["last_update"][:] = kf
    split = np.array([[kf, 0, 1], [kf, 1, len(store) - 1]], np.int32)
    ctx.inactive_load(s, split)
    assert ctx.inactive_segments().tolist() == split.tolist() and ctx.inactive_download(kf).tobytes() == s.tobytes()
    ctx.inactive_load(s[:0], split[:0])
    assert ctx.inactive_size() == (0, 0)
    for c in (ctx, big, none):
        c.close()


def test_save_after_a_rejected_frame_and_into_an_unwritable_directory(tmp_path):
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    a = new_ctx(store=STORE)
    run(a, lists, 0, first, 1)
    b = new_ctx(store=1)                                  # the first retirement does not fit
    windowed(b, 0, first + 2, lists, want_counts=False)
    path = tmp_path / "map.dsm"
    with pytest.raises(capi.DsmError) as e:
        b.map_save(str(path))
    assert e.value.code == -6 and not path.exists() and os.listdir(tmp_path) == []
    b.map_save(str(path))                                 # cleared: the map of the last applied frame
    _, pool, store, table, _, ok = parse(path.read_bytes())
    assert ok and pool.tobytes() == a.pool_download().tobytes() and len(store) == 0
    for d in (tmp_path / "missing" / "map.dsm",):
        with pytest.raises(capi.DsmError) as e:
            a.map_save(str(d))
        assert e.value.code == -9 and not d.exists()
    ro = tmp_path / "ro"
    ro.mkdir()
    ro.chmod(0o500)
    try:
        if not os.access(ro, os.W_OK):                    # not meaningful for a user who may write anywhere
            with pytest.raises(capi.DsmError) as e:
                a.map_save(str(ro / "map.dsm"))
            assert e.value.code == -9 and os.listdir(ro) == []
    finally:
        ro.chmod(0o700)
    a.close()
    b.close()


@pytest.mark.parametrize("chunk", [1, 4])
def test_publishing_after_a_load(tmp_path, chunk):
    lists = simple_lists()
    a = new_ctx(store=STORE)
    run(a, lists, 0, 10, chunk)
    path = str(tmp_path / "map.dsm")
    a.map_save(path)
    b = new_ctx(store=STORE)
    b.publish_enable()
    run(b, lists, 0, 3, 1)
    snapshot_equals_readers(b, Mirror(), "before the load")
    b.map_load(path)
    mirror = Mirror()                                     # the load reset the host's view: everything is forwarded
    _, inactive, cf = snapshot_equals_readers(b, mirror, "first snapshot after the load")
    assert cf == 0 and len(inactive) > 0
    assert b.publish_chunks() == -(-len(inactive) // 256)
    for s in range(10, T, chunk):
        for c in (a, b):
            windowed(c, s, min(T, s + chunk), lists, want_counts=False)
        snapshot_equals_readers(b, mirror, f"frames from {s}")
        assert_same(a, b, f"frames from {s}")
    a.close()
    b.close()


# ---- the node ----
N_NODE = 24


def run_checkpoint_main(tmp, cam, script, drift_free_poses, j):
    from test_cpp_adapter import build_adapter
    exe = build_adapter("checkpoint_main")
    fin, fout, ckpt = os.path.join(tmp, "script.bin"), os.path.join(tmp, "out.bin"), os.path.join(tmp, "node.dsm")
    with open(fin, "wb") as f:
        f.write(bytes(script.b))
    args = [exe, str(cam.width), str(cam.height)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]
    r = subprocess.run(args + [str(drift_free_poses), str(j), ckpt, fin, fout, tmp], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return np.frombuffer(open(fout, "rb").read(), np.int32)


# j: messages fed before the save (three per frame: orb, image, depth); frame 16's orb message brings the first loop
# correction that moves every pose, frame 9's a loop edge back to keyframe 0
@pytest.mark.parametrize("drift_free_poses,j", [(1, 3 * 7 + 1), (1, 3 * 16 + 1), (1, 3 * 11 + 2), (10, 3 * 9 + 2),
                                                (10, 3 * 16 + 1), (2, 3 * 13 + 3)])
def test_node_resumes_from_its_checkpoint(tmp_path, drift_free_poses, j):
    cam = synth.KITTI
    msgs = drive(N_NODE)
    sc = Script()
    for t, (stamp, is_kf, ref, p7, path, loops) in enumerate(msgs):
        sc.orb(stamp, is_kf, ref, p7, path, loops)
        sc.images(stamp, *synth.make_frame(cam, 3000 + t, synth.pose_stream(t)))
    out = run_checkpoint_main(str(tmp_path), cam, sc, drift_free_poses, j).tolist()
    n_rest = 3 * N_NODE - j
    assert len(out) == 3 + 3 * n_rest + 5
    assert out[:3] == [0, 0, 1], "save, load, equal right after the load"
    for m in range(n_rest):
        ra, rb, same = out[3 + 3 * m: 6 + 3 * m]
        assert ra == rb == 0 and same == 1, f"message {j + m}: node A {ra}, node B {rb}, equal {same}"
    tail = out[3 + 3 * n_rest:]
    assert tail[:2] == [-1, 1], "a node with other parameters refuses the file and is unchanged"
    assert tail[2:4] == [-1, 1], "a file without a node section is refused and the node is unchanged"
    assert tail[4] == 0
    for a, b in (("a.ply", "b.ply"), ("a.pcd", "b.pcd")):
        assert open(tmp_path / a, "rb").read() == open(tmp_path / b, "rb").read(), a
    assert os.path.getsize(tmp_path / "a.ply") > 1000
