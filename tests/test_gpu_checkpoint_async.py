"""Checkpoints that do not stop the stream (dsm_checkpoint_enable / _enqueue / _wait, DESIGN.md §8.5).

The file is byte for byte what dsm_map_save writes at the enqueue's position in the stream, whatever the context does
while it drains: further frames, reactivations that compact the store under the snapshot, loop-closure warps, a publish
snapshot.  Checkpoints leave the map exactly as a drive without them; a fresh context resumes from the file; the error
and call-sequence contract; and dsm::SurfelMapNode's save_state_async (tests/cpp/checkpoint_async_main.cpp)."""
import ctypes
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from checkpoint_files import parse
from node_drive import node_script, run_driver
from resident_map import SAVES, STORE, T, frames, loop_warp, made, new_ctx, readers, run, simple_lists, stored_keyframes, windowed
from util import CAM

pytestmark = pytest.mark.gpu

DSM_E_CAPACITY, DSM_E_STATE, DSM_E_IO = -6, -7, -9


def async_ctx(constants="drive", **kw):
    ctx = made(constants, **kw)
    ctx.checkpoint_enable()
    return ctx


@pytest.mark.parametrize("save", sorted(SAVES))
@pytest.mark.parametrize("chunk", [1, 4, 8])
@pytest.mark.parametrize("constants", ["drive", "rgbd"])
def test_the_file_is_map_save_at_the_enqueue(tmp_path, save, chunk, constants):
    """A enqueues at the save point and fuses every remaining frame before it waits; B stops there and saves."""
    lists = simple_lists()
    k, when = SAVES[save]
    a, b = async_ctx(constants, store=STORE), made(constants, store=STORE)
    for c in (a, b):
        run(c, lists, 0, k, chunk)
    if when == "before":
        kfs = stored_keyframes(b)
        loop_warp(a, kfs)
        loop_warp(b, kfs)
    pa, pb = tmp_path / "async.dsm", tmp_path / "sync.dsm"
    a.checkpoint_enqueue(str(pa), extra=b"node")
    if when == "after":
        loop_warp(a, stored_keyframes(b))
    run(a, lists, k, T, chunk)
    assert a.checkpoint_wait()
    b.map_save(str(pb), extra=b"node")
    assert pa.read_bytes() == pb.read_bytes()
    assert sorted(os.listdir(tmp_path)) == ["async.dsm", "sync.dsm"]      # no temporary left behind
    a.close()
    b.close()


def test_reactivations_and_warps_under_the_snapshot(tmp_path):
    """Enqueued at frame 5; A then runs through both reactivations (frames 9 and 13, which compact the store the snapshot
    was taken from) and a loop closure on the pool and every stored keyframe, all before the wait."""
    lists = simple_lists()
    assert lists[9][2] and lists[13][2]
    a, b = async_ctx(store=STORE), made(store=STORE)
    for c in (a, b):
        run(c, lists, 0, 5, 1)
    kfs = stored_keyframes(b)
    assert kfs
    a.checkpoint_enqueue(str(tmp_path / "a.dsm"))
    run(a, lists, 5, 11, 3)
    loop_warp(a, kfs)
    run(a, lists, 11, T, 1)
    loop_warp(a, [0, 1])
    assert a.checkpoint_wait()
    b.map_save(str(tmp_path / "b.dsm"))
    assert (tmp_path / "a.dsm").read_bytes() == (tmp_path / "b.dsm").read_bytes()
    h, pool, store, table, extra, ok = parse((tmp_path / "a.dsm").read_bytes())
    assert ok and len(store) > 0 and len(table) > 0
    a.close()
    b.close()


@pytest.mark.parametrize("chunk,every", [(1, 2), (4, 1), (8, 1)])
def test_checkpoints_leave_the_map_as_a_drive_without_them(tmp_path, chunk, every):
    """A checkpoint every `every` calls, polled without blocking on the next calls: pool, store, table and both clouds
    equal the same drive without checkpoints after every call, and every file equals the twin's dsm_map_save."""
    lists = simple_lists()
    a, b = async_ctx(store=STORE), made(store=STORE)
    pending, written = None, 0
    for i, s in enumerate(range(0, T, chunk)):
        for c in (a, b):
            run(c, lists, s, min(T, s + chunk), chunk)
        if pending and a.checkpoint_wait(block=False):
            pending = None
            written += 1
        if i % every == 0:
            if pending:
                assert a.checkpoint_wait()
                written += 1
            p = tmp_path / f"{i}.dsm"
            a.checkpoint_enqueue(str(p), extra=bytes([i]))
            b.map_save(str(tmp_path / f"{i}.want"), extra=bytes([i]))
            pending = p
        assert readers(a) == readers(b), f"frames {s}-{min(T, s + chunk) - 1}"
    if pending:
        assert a.checkpoint_wait()
        written += 1
    names = sorted(n for n in os.listdir(tmp_path) if n.endswith(".dsm"))
    assert written == len(names) > 0
    for n in names:
        assert (tmp_path / n).read_bytes() == (tmp_path / n.replace(".dsm", ".want")).read_bytes(), n
    a.close()
    b.close()


@pytest.mark.parametrize("k", [10, 14])
def test_resume_from_the_async_file(tmp_path, k):
    lists = simple_lists()
    a, ref = async_ctx(store=STORE), made(store=STORE)
    for c in (a, ref):
        run(c, lists, 0, k, 4)
    path = str(tmp_path / "map.dsm")
    a.checkpoint_enqueue(path, extra=b"resume")
    run(a, lists, k, T, 4)
    assert a.checkpoint_wait()
    b = made(store=STORE)
    assert b.map_load(path) == b"resume"
    assert readers(b) == readers(ref)
    for s in range(k, T, 2):
        for c in (b, ref):
            run(c, lists, s, min(T, s + 2), 2)
        assert readers(b) == readers(ref), f"frames from {s}"
    assert readers(a) == readers(ref)
    for c in (a, b, ref):
        c.close()


def test_a_rejected_frame_writes_no_file_and_leaves_the_error(tmp_path):
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    b = new_ctx(store=1)                                  # the first retirement does not fit
    b.checkpoint_enable()
    windowed(b, 0, first + 2, lists, want_counts=False)
    path = tmp_path / "map.dsm"
    b.checkpoint_enqueue(str(path))
    with pytest.raises(capi.DsmError) as e:
        b.checkpoint_wait()
    assert e.value.code == DSM_E_CAPACITY and os.listdir(tmp_path) == []
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()                                     # the next synchronising reader reports and clears it
    assert e.value.code == DSM_E_CAPACITY
    a = new_ctx(store=STORE)
    run(a, lists, 0, first, 1)
    assert b.pool_download().tobytes() == a.pool_download().tobytes()
    b.checkpoint_enqueue(str(path))                       # cleared: the map of the last applied frame
    assert b.checkpoint_wait()
    _, pool, store, _, _, ok = parse(path.read_bytes())
    assert ok and pool.tobytes() == a.pool_download().tobytes() and len(store) == 0
    a.close()
    b.close()


def test_an_unwritable_path_leaves_nothing(tmp_path):
    lists = simple_lists()
    a = async_ctx(store=STORE)
    run(a, lists, 0, 6, 3)
    missing = tmp_path / "missing" / "map.dsm"
    a.checkpoint_enqueue(str(missing))
    with pytest.raises(capi.DsmError) as e:
        a.checkpoint_wait()
    assert e.value.code == DSM_E_IO and not missing.exists() and os.listdir(tmp_path) == []
    ro = tmp_path / "ro"
    ro.mkdir()
    ro.chmod(0o500)
    try:
        if not os.access(ro, os.W_OK):                    # not meaningful for a user who may write anywhere
            a.checkpoint_enqueue(str(ro / "map.dsm"))
            with pytest.raises(capi.DsmError) as e:
                a.checkpoint_wait()
            assert e.value.code == DSM_E_IO and os.listdir(ro) == []
    finally:
        ro.chmod(0o700)
    a.checkpoint_enqueue(str(tmp_path / "map.dsm"))      # the failed writes were retired
    assert a.checkpoint_wait()
    a.close()


def test_call_sequence_errors(tmp_path):
    L = capi.load_library()
    p = os.fsencode(tmp_path / "map.dsm")
    fin = ctypes.c_int(7)
    bare = capi.Context(CAM, max_batch=1, max_local_surfels=1 << 16)
    assert L.dsm_checkpoint_enable(bare.h) == DSM_E_STATE                 # no resident pool
    bare.close()
    ctx = new_ctx(store=STORE)
    assert L.dsm_checkpoint_enqueue(ctx.h, p, None, 0) == DSM_E_STATE     # before enable
    assert L.dsm_checkpoint_wait(ctx.h, 1, ctypes.byref(fin)) == DSM_E_STATE and fin.value == 0
    ctx.checkpoint_enable()
    assert L.dsm_checkpoint_enable(ctx.h) == DSM_E_STATE                  # once
    assert L.dsm_checkpoint_wait(ctx.h, 0, ctypes.byref(fin)) == DSM_E_STATE   # nothing enqueued
    assert L.dsm_checkpoint_enqueue(ctx.h, None, None, 0) == -1
    assert L.dsm_checkpoint_enqueue(ctx.h, p, None, 4) == -1
    run(ctx, simple_lists(), 0, 4, 4)
    ctx.checkpoint_enqueue(str(tmp_path / "map.dsm"))
    assert L.dsm_checkpoint_enqueue(ctx.h, p, None, 0) == DSM_E_STATE     # the first is not retired
    assert L.dsm_inactive_reserve(ctx.h, STORE) == DSM_E_STATE            # its images are sized by the store
    assert L.dsm_debug_checkpoint_drain_ctas(ctx.h, 8) == DSM_E_STATE
    assert ctx.checkpoint_wait()
    assert L.dsm_checkpoint_wait(ctx.h, 1, ctypes.byref(fin)) == DSM_E_STATE   # retired
    assert os.listdir(tmp_path) == ["map.dsm"]
    ctx.close()


def test_no_checkpoint_of_a_batch_buffer(tmp_path):
    """A batch call leaves its slices in the pool buffer and no resident pool: like dsm_map_save, the enqueue is refused
    and the last good checkpoint under the path stays as it was, until dsm_pool_upload makes a pool resident again."""
    lists = simple_lists()
    a = async_ctx(store=STORE)
    run(a, lists, 0, 6, 3)
    path = tmp_path / "map.dsm"
    a.checkpoint_enqueue(str(path))
    assert a.checkpoint_wait()
    good = path.read_bytes()
    pose, gray, depth = frames()[0]
    a.fuse_frame(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))   # a batch call on the same context
    with pytest.raises(capi.DsmError) as e:
        a.map_save(str(tmp_path / "sync.dsm"))
    assert e.value.code == DSM_E_STATE
    L = capi.load_library()
    assert L.dsm_checkpoint_enqueue(a.h, os.fsencode(path), None, 0) == DSM_E_STATE
    assert L.dsm_checkpoint_wait(a.h, 1, None) == DSM_E_STATE       # nothing was enqueued
    assert path.read_bytes() == good and os.listdir(tmp_path) == ["map.dsm"]
    b = made(store=STORE)
    run(b, lists, 0, 6, 3)
    a.pool_upload(b.pool_download())                                 # resident again
    a.checkpoint_enqueue(str(path))
    assert a.checkpoint_wait()
    b.map_save(str(tmp_path / "want.dsm"))
    assert path.read_bytes() == (tmp_path / "want.dsm").read_bytes()
    a.close()
    b.close()


def test_reserve_rebuilds_the_images(tmp_path):
    lists = simple_lists()
    a, b = async_ctx(store=0), made(store=0)
    for c in (a, b):
        c.inactive_reserve(STORE // 2)                    # after enable: the images follow the new reservation
        run(c, lists, 0, 8, 4)
    a.checkpoint_enqueue(str(tmp_path / "a.dsm"))
    b.map_save(str(tmp_path / "b.dsm"))
    assert a.checkpoint_wait()
    assert (tmp_path / "a.dsm").read_bytes() == (tmp_path / "b.dsm").read_bytes()
    # without a store: an empty store section
    c, d = async_ctx(store=0), made(store=0)
    for x in (c, d):
        windowed(x, 0, 3, lists, want_counts=False, empty=True)
    c.checkpoint_enqueue(str(tmp_path / "c.dsm"))
    d.map_save(str(tmp_path / "d.dsm"))
    assert c.checkpoint_wait()
    assert (tmp_path / "c.dsm").read_bytes() == (tmp_path / "d.dsm").read_bytes()
    for x in (a, b, c, d):
        x.close()


def test_destroy_finishes_a_pending_write(tmp_path):
    lists = simple_lists()
    a, b = async_ctx(store=STORE), made(store=STORE)
    for c in (a, b):
        run(c, lists, 0, 12, 4)
    path = tmp_path / "map.dsm"
    a.checkpoint_enqueue(str(path), extra=b"last")
    run(a, lists, 12, T, 4)
    a.close()                                             # returns once the file is complete
    assert capi.map_peek(path)[0] == b"last"
    b.map_save(str(tmp_path / "want.dsm"), extra=b"last")
    assert path.read_bytes() == (tmp_path / "want.dsm").read_bytes()
    b.close()


def test_a_publish_snapshot_and_a_checkpoint_in_flight_together(tmp_path):
    lists = simple_lists()
    a, b = async_ctx(store=STORE), made(store=STORE)
    a.publish_enable()
    for c in (a, b):
        run(c, lists, 0, 9, 3)
    a.publish_enqueue(5)
    a.checkpoint_enqueue(str(tmp_path / "a.dsm"))
    run(a, lists, 9, T, 1)
    active, inactive, _ = a.publish_wait()
    assert active.tobytes() == b.pool_export_cloud(5).tobytes()
    assert inactive.tobytes() == b.inactive_export_cloud().tobytes()
    assert a.checkpoint_wait()
    b.map_save(str(tmp_path / "b.dsm"))
    assert (tmp_path / "a.dsm").read_bytes() == (tmp_path / "b.dsm").read_bytes()
    a.close()
    b.close()


# ---- the node ----
N_NODE = 24


# j: messages fed before the save (three per frame: orb, image, depth), the save points of test_gpu_checkpoint.py's node
@pytest.mark.parametrize("drift_free_poses,j", [(1, 3 * 7 + 1), (1, 3 * 16 + 1), (10, 3 * 9 + 2), (2, 3 * 13 + 3)])
def test_node_save_state_async(tmp_path, drift_free_poses, j):
    cam = synth.KITTI
    sc = node_script(cam, N_NODE)
    args = [drift_free_poses, j, tmp_path / "a.dsm", tmp_path / "t.dsm"]
    out = run_driver("checkpoint_async_main", str(tmp_path), cam, sc, args, after=[tmp_path]).take(np.int32, -1).tolist()
    n_rest = 3 * N_NODE - j
    assert len(out) == 3 + n_rest + 4 + 3 * n_rest + 2
    assert out[:3] == [0, 0, 0], "enable, save_state_async, twin's save_state"
    assert out[3:3 + n_rest] == [0] * n_rest, "node A while its checkpoint is written"
    o = 3 + n_rest
    assert out[o] == 0 and 1 <= out[o + 1] <= n_rest, "the write, and the messages A received meanwhile"
    assert (tmp_path / "a.dsm").read_bytes() == (tmp_path / "t.dsm").read_bytes(), "save_state_async equals save_state"
    assert out[o + 2:o + 4] == [0, 1], "load, equal right after the load"
    o += 4
    for m in range(n_rest):
        rb, rt, same = out[o + 3 * m: o + 3 * m + 3]
        assert rb == rt == 0 and same == 1, f"message {j + m}: node B {rb}, twin {rt}, equal {same}"
    o += 3 * n_rest
    assert out[o:] == [1, 0], "A, which kept going while it saved, equals the twin; the files were written"
    for x in ("ply", "pcd"):
        want = (tmp_path / f"t.{x}").read_bytes()
        assert (tmp_path / f"a.{x}").read_bytes() == want and (tmp_path / f"b.{x}").read_bytes() == want, x
    assert os.path.getsize(tmp_path / "t.ply") > 1000
