"""dsm_publish_enable / _enqueue / _wait: the node's active and inactive clouds from inside the stream.

The snapshot equals the synchronous readers (dsm_pool_export_cloud, dsm_inactive_export_cloud) byte for byte at its
position in the stream; inactive_changed_from and the number of forwarded chunks equal the chunk rule restated in
oracle/pyoracle_publish.py; the error contract; and dsm::SurfelMapNode::published_clouds (tests/cpp/publish_main.cpp)."""

import numpy as np
import pytest

import pyoracle_publish
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import (
    Mirror, STORE, T, needs_window_oracle, new_ctx, node_lists, simple_lists, snapshot_equals_readers, warp, windowed)
from util import CAM

pytestmark = pytest.mark.gpu


def run_drive(lists, chunk):
    ctx = new_ctx(store=STORE)
    ctx.publish_enable()
    mirror = Mirror()
    stored, seen = set(), {"retire_only": 0, "grew": 0, "shrank": 0, "warped": 0}
    for t0 in range(0, T, chunk):
        t1 = min(T, t0 + chunk)
        windowed(ctx, t0, t1, lists, want_counts=False)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        warped = False
        if (t0 // chunk) % 2 == 1 and stored:   # a loop closure between two calls: the pool and one stored keyframe move
            ctx.pool_transform(warp(1))
            ctx.inactive_transform(max(stored), warp(2))
            warped = True
        prev = mirror.prev
        what = f"after frames {t0}-{t1 - 1}"
        _, inactive, cf = snapshot_equals_readers(ctx, mirror, what)
        n = len(inactive)
        seen["grew"] += n > prev
        seen["shrank"] += n < prev
        seen["warped"] += warped
        if chunk == 1 and not warped and lists[t0][1] and not lists[t0][2]:
            assert cf == prev, f"{what}: a retire-only frame changes nothing below the previous size"
            seen["retire_only"] += 1
        # nothing happened since: the same inactive cloud, no chunk crosses; the other filter of the active cloud
        a1, i1, cf1 = snapshot_equals_readers(ctx, mirror, what + ", again", min_update_times=1)
        assert ctx.publish_chunks() == 0 and cf1 == n and i1.tobytes() == inactive.tobytes()
    assert seen["grew"] and seen["warped"], seen
    ctx.close()
    return seen


@needs_window_oracle
@pytest.mark.parametrize("chunk", [1, 3, 8])
@pytest.mark.parametrize("drift_free_poses", [1, 2, 10])
def test_snapshot_equals_the_synchronous_readers_on_the_node_drives(drift_free_poses, chunk):
    if drift_free_poses == 10:   # nothing leaves a window of 10 in 16 frames: the store stays empty
        lists = node_lists(drift_free_poses)
        ctx = new_ctx(store=STORE)
        ctx.publish_enable()
        mirror = Mirror()
        for t0 in range(0, T, chunk):
            windowed(ctx, t0, min(T, t0 + chunk), lists, want_counts=False)
            snapshot_equals_readers(ctx, mirror, f"after frames from {t0}")
        ctx.close()
        return
    seen = run_drive(node_lists(drift_free_poses), chunk)
    if chunk == 1:
        assert seen["retire_only"] and (seen["shrank"] or drift_free_poses != 2), seen


@pytest.mark.parametrize("chunk", [1, 3, 8])
def test_snapshot_equals_the_synchronous_readers(chunk):
    seen = run_drive(simple_lists(), chunk)
    if chunk == 1:
        assert seen["retire_only"] and seen["shrank"], seen


def test_changed_from_of_a_warped_keyframe_and_of_a_reactivation():
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    ctx.publish_enable()
    mirror = Mirror()
    windowed(ctx, 0, 9, lists, want_counts=False)
    _, before, _ = snapshot_equals_readers(ctx, mirror, "after frames 0-8")
    store = ctx.inactive_download(-1)
    kf = 1
    own = np.nonzero(store["last_update"] == kf)[0]
    assert len(own) and own[0] > 0, "keyframe 1 holds a segment that is not the first"
    ctx.inactive_transform(kf, warp(3))
    _, after, cf = snapshot_equals_readers(ctx, mirror, "after the warp of keyframe 1")
    assert cf == own[0], "the warped keyframe's first segment offset"
    diff = (after.view(np.uint32).reshape(-1, 4) != before.view(np.uint32).reshape(-1, 4)).any(1)
    assert ctx.publish_chunks() == len(set((np.nonzero(diff)[0] // pyoracle_publish.CHUNK).tolist()))
    # frame 9 reactivates keyframe 0, the first segment: everything above moves down
    assert (store["last_update"][0] == 0) and lists[9][2] == [0]
    windowed(ctx, 9, 10, lists, want_counts=False)
    _, moved, cf = snapshot_equals_readers(ctx, mirror, "after the reactivation of keyframe 0")
    assert cf == 0 and len(moved) == len(after) - int((store["last_update"] == 0).sum())
    ctx.close()


def test_stream_order_without_synchronising():
    """fuse A, publish, fuse B, never waiting in between: the snapshot is the map after A."""
    lists = simple_lists()
    a, b = new_ctx(max_batch=16, store=STORE), new_ctx(max_batch=16, store=STORE)
    a.publish_enable()
    windowed(a, 0, 8, lists, want_counts=False)
    a.publish_enqueue(5)
    windowed(a, 8, 16, lists, want_counts=False)
    active, inactive, cf = a.publish_wait()
    windowed(b, 0, 8, lists, want_counts=False)
    assert active.tobytes() == b.pool_export_cloud(5).tobytes()
    assert inactive.tobytes() == b.inactive_export_cloud().tobytes()
    assert cf == 0 and len(inactive) > 0
    windowed(b, 8, 16, lists, want_counts=False)
    assert a.pool_download().tobytes() == b.pool_download().tobytes()       # and the snapshot disturbed nothing
    assert a.inactive_export_cloud().tobytes() != inactive.tobytes()
    a.close()
    b.close()


def test_pipelined_one_frame_late():
    """The snapshot of frame t-1 is collected at the start of frame t: every snapshot equals the synchronous export of
    its frame in a replay."""
    lists = simple_lists()
    ctx = new_ctx(max_batch=2, store=STORE)
    ctx.publish_enable()
    snaps = []
    for t in range(T):
        if t:
            snaps.append(ctx.publish_wait())
        windowed(ctx, t, t + 1, lists, want_counts=False)
        if t == 10:
            ctx.inactive_transform(2, warp(2))   # a loop closure lands between the fuse and its snapshot
        ctx.publish_enqueue(5)
    snaps.append(ctx.publish_wait())
    ctx.close()
    replay = new_ctx(max_batch=2, store=STORE)
    shadow, prev = np.zeros((STORE, 4), np.float32), 0
    for t, (active, inactive, cf) in enumerate(snaps):
        windowed(replay, t, t + 1, lists, want_counts=False)
        if t == 10:
            replay.inactive_transform(2, warp(2))
        assert active.tobytes() == replay.pool_export_cloud(5).tobytes(), f"frame {t}: active cloud"
        assert inactive.tobytes() == replay.inactive_export_cloud().tobytes(), f"frame {t}: inactive cloud"
        _, want, shadow = pyoracle_publish.mirror_step(shadow, prev, inactive.view(np.float32).reshape(-1, 4))
        assert cf == want, f"frame {t}: inactive_changed_from"
        prev = len(inactive)
    replay.close()


def test_call_sequence_errors_and_no_store():
    lib = capi.load_library()
    bare = capi.Context(CAM, max_batch=1, max_local_surfels=1 << 16)
    assert lib.dsm_publish_enable(bare.h) == -7          # no resident pool
    bare.close()
    ctx = new_ctx(store=0)
    assert lib.dsm_publish_enqueue(ctx.h, 5) == -7       # before enable
    assert lib.dsm_publish_wait(ctx.h, None, None, None, None, None) == -7
    ctx.publish_enable()
    assert lib.dsm_publish_enable(ctx.h) == -7           # once
    assert lib.dsm_publish_wait(ctx.h, None, None, None, None, None) == -7   # nothing enqueued
    windowed(ctx, 0, 8, simple_lists(), want_counts=False, empty=True)
    ctx.publish_enqueue(5)
    assert lib.dsm_publish_enqueue(ctx.h, 5) == -7       # one snapshot in flight
    assert lib.dsm_inactive_reserve(ctx.h, 1000) == -7   # nor may its buffers be rebuilt
    active, inactive, cf = ctx.publish_wait()
    assert len(inactive) == 0 and cf == 0                # no store reserved
    assert len(active) > 0 and active.tobytes() == ctx.pool_export_cloud(5).tobytes()
    assert lib.dsm_publish_wait(ctx.h, None, None, None, None, None) == -7
    ctx.publish_enqueue(1)
    assert lib.dsm_publish_wait(ctx.h, None, None, None, None, None) == 0    # every out-pointer may be NULL
    ctx.close()


def test_reserve_after_enable_rebuilds_the_mirror():
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    ctx.publish_enable()
    mirror = Mirror()
    windowed(ctx, 0, 7, lists, want_counts=False)
    _, inactive, _ = snapshot_equals_readers(ctx, mirror, "after frames 0-6")
    assert len(inactive) > 0
    kfs = sorted(set(ctx.inactive_download(-1)["last_update"].tolist()))
    for kf in kfs:
        ctx.inactive_reactivate(kf)
    assert ctx.inactive_size()[0] == 0
    ctx.inactive_reserve(STORE // 2)
    assert ctx.inactive_retire(kfs[0]) > 0
    fresh = Mirror(STORE // 2)
    _, inactive, cf = snapshot_equals_readers(ctx, fresh, "after the new reservation")
    assert cf == 0 and len(inactive) > 0
    ctx.close()


def test_store_overflow_comes_back_from_wait_and_stays_for_the_next_read():
    """The drive of a store too small: the frame that would overflow it is not applied; the snapshot holds the map of
    the last applied frame and returns DSM_E_CAPACITY; the next synchronising call still reports and clears it."""
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    a = new_ctx(store=STORE)
    windowed(a, 0, first, lists, want_counts=False)
    b = new_ctx(store=1)
    b.publish_enable()
    windowed(b, 0, first + 2, lists, want_counts=False)
    b.publish_enqueue(1)
    with pytest.raises(capi.DsmError) as e:
        b.publish_wait()
    assert e.value.code == -6
    active, inactive, cf = e.value.clouds
    assert active.tobytes() == a.pool_export_cloud(1).tobytes() and len(active) > 0
    assert len(inactive) == 0
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    assert b.pool_size() == a.pool_size()
    b.publish_enqueue(1)
    active2, _, _ = b.publish_wait()                     # cleared: an ordinary snapshot again
    assert active2.tobytes() == active.tobytes()
    a.close()
    b.close()


def test_publisher_that_never_synchronises_past_the_capacity():
    """A publisher never refreshes the host's bound of the pool size, which grows by one frame of seeds per fused
    frame: here it passes the capacity several times over (112 frames of 1200 seeds on a pool of 32 Ki).  The launches
    stay sized by the capacity, and every snapshot equals the readers of a twin context that synchronises after every
    call."""
    from densesurfelmapping_b200.elements import num_seeds
    lists = simple_lists()
    cap, chunk, passes = 1 << 15, 8, 7
    assert passes * T * num_seeds(CAM.width, CAM.height) > 4 * cap
    ctx, twin = new_ctx(cap=cap, store=STORE), new_ctx(cap=cap, store=STORE)
    ctx.publish_enable()
    for k in range(passes):
        for t0 in range(0, T, chunk):
            for c in (ctx, twin):
                windowed(c, t0, t0 + chunk, lists, want_counts=False, empty=k > 0)
            ctx.publish_enqueue(5)           # the context under test is never read synchronously
            active, inactive, _ = ctx.publish_wait()
            what = f"pass {k}, frames {t0}-{t0 + chunk - 1}"
            assert active.tobytes() == twin.pool_export_cloud(5).tobytes(), f"{what}: active cloud"
            assert inactive.tobytes() == twin.inactive_export_cloud().tobytes(), f"{what}: inactive cloud"
    assert len(active) > 0 and len(inactive) > 0
    assert ctx.pool_download().tobytes() == twin.pool_download().tobytes()
    assert ctx.inactive_download(-1).tobytes() == twin.inactive_download(-1).tobytes()
    ctx.close()
    twin.close()


# ---- the node ----
@pytest.mark.parametrize("drift_free_poses", [1, 2])
def test_node_publishes_what_its_readers_return(tmp_path, drift_free_poses):
    cam, n = synth.KITTI, 30
    sc = node_script(cam, n)
    r = run_driver("publish_main", str(tmp_path), cam, sc, [drift_free_poses, 0, 1 << 20, 1 << 21, 1], tag=1)
    prev, warped = np.zeros(0, POINT_DTYPE), 0
    for t in range(n):
        rc, cf = r.i(), r.i()
        active, inactive = r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        assert rc == 0 and r.i() == 0, f"frame {t}"
        assert active.tobytes() == r.lst(POINT_DTYPE).tobytes(), f"frame {t}: active cloud"
        assert inactive.tobytes() == r.lst(POINT_DTYPE).tobytes(), f"frame {t}: inactive cloud"
        m = min(len(prev), len(inactive))
        diff = np.nonzero((prev[:m].view(np.uint32).reshape(-1, 4) != inactive[:m].view(np.uint32).reshape(-1, 4)).any(1))[0]
        want = int(diff[0]) if len(diff) else m
        assert cf == want, f"frame {t}: inactive_changed_from"
        warped += len(diff) > 0
        prev = inactive.copy()
    end = (r.lst(SURFEL_DTYPE).tobytes(), r.lst(POINT_DTYPE).tobytes())
    assert r.o == len(r.raw) and len(prev) > 0 and warped > 0
    q = run_driver("publish_main", str(tmp_path), cam, sc, [drift_free_poses, 0, 1 << 20, 1 << 21, 0], tag=0)
    assert (q.lst(SURFEL_DTYPE).tobytes(), q.lst(POINT_DTYPE).tobytes()) == end, "publishing perturbed the map"
    assert q.o == len(q.raw)
