"""GPU-resident pool mode (SURVEY.md §8f rows 1-2): device-side post-fusion compaction/append and the
loop-closure pool transform, against the restated caller-side steps of SurfelMap."""
import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import check_surfels, oracle_for

pytestmark = pytest.mark.gpu


def match_as_sets(got, want, tol=1e-4):
    """Pools are equal as sets: same size, and a one-to-one nearest-neighbour matching within tolerance."""
    assert len(got) == len(want), f"pool size {len(got)} != {len(want)}"
    if len(got) == 0:
        return
    key = lambda a: np.lexsort((a["pz"], a["py"], a["px"], a["last_update"], a["update_times"]))
    g, w = got[key(got)], want[key(want)]
    # lexsort on floats can differ in the last bits; repair by nearest neighbour inside equal-integer groups
    pg = np.stack([g["px"], g["py"], g["pz"]], -1).astype(np.float64)
    pw = np.stack([w["px"], w["py"], w["pz"]], -1).astype(np.float64)
    bad = np.nonzero(np.linalg.norm(pg - pw, axis=1) > tol * np.maximum(np.linalg.norm(pw, axis=1), 1.0))[0]
    if len(bad):
        used = set()
        for i in bad:
            dist = np.linalg.norm(pw[bad] - pg[i], axis=1)
            j = int(np.argmin(dist))
            assert dist[j] <= tol * max(np.linalg.norm(pg[i]), 1.0) and j not in used, f"surfel {i} has no partner"
            used.add(j)
            g[i], w_i = g[i], w[bad[j]]
            check_surfels(g[i:i + 1], np.array([w_i]), "set member")
        ok = np.setdiff1d(np.arange(len(g)), bad)
        check_surfels(g[ok], w[ok], "pool (sorted)")
    else:
        check_surfels(g, w, "pool (sorted)")


def test_resident_stream_matches_reference_flow():
    """Per frame: hot path on the resident pool + device compaction/append == oracle fuse + fuse_map post-step."""
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=100000)
    orc = oracle_for(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    ctx.pool_upload(pool)
    for t in range(4):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 300 + t, pose)
        lo, no = orc.fuse(t // 2 + (7 if t == 3 else 0), gray, depth, pose, pool)  # the jump in ref idx kills unstable surfels
        want = pyoracle.fuse_map_poststep(lo, no)
        ctx.pool_upload(pool)  # re-sync to the oracle's pool so one tolerance-sized drift cannot flip a decision later
        n_new = ctx.fuse_frame_resident(t // 2 + (7 if t == 3 else 0), gray, depth, pose, want_count=True)
        assert n_new == len(no)
        got = ctx.pool_download()
        match_as_sets(got, want)
        assert (got["update_times"] > 0).all()
        pool = want
    assert (lo["update_times"] == 0).sum() > 0, "test never exercised the kill path"
    ctx.close()


def test_resident_stream_free_running():
    """No re-sync: 6 frames carried entirely on the device stay within tolerance of the oracle flow."""
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=100000)
    orc = oracle_for(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    ctx.pool_upload(pool)
    for t in range(6):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 400 + t, pose)
        lo, no = orc.fuse(t // 2, gray, depth, pose, pool)
        pool = pyoracle.fuse_map_poststep(lo, no)
        ctx.fuse_frame_resident(t // 2, gray, depth, pose)
    got = ctx.pool_download()
    assert abs(len(got) - len(pool)) <= max(2, len(pool) // 500)
    if len(got) == len(pool):
        match_as_sets(got, pool, tol=1e-3)
    ctx.close()


def test_pool_transform_loop_closure():
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    gray, depth = synth.make_frame(cam, 0)
    orc = oracle_for(cam)
    _, pool = orc.fuse(0, gray, depth, synth.identity_pose(), np.zeros(0, SURFEL_DTYPE))
    a = np.deg2rad(2.0)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    Wm[:3, 3] = [0.5, -0.1, 0.25]
    w = np.ascontiguousarray(Wm.T.astype(np.float32).reshape(16))
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=len(pool) + 10)
    ctx.pool_upload(pool)
    ctx.pool_transform(w)
    got = ctx.pool_download()
    check_surfels(got, pyoracle.warp_active(pool, w), "warped pool")
    ctx.close()


def test_pool_retire_and_append_move_add_surfels():
    """move_add_surfels on the resident pool (surfel_map.cpp:1479-1497, :1583-1587): exact, ordered."""
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    orc = oracle_for(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    for t in range(3):  # a pool whose surfels carry last_update in {0, 1, 2}
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 500 + t, pose)
        lo, no = orc.fuse(t, gray, depth, pose, pool)
        pool = pyoracle.fuse_map_poststep(lo, no)
    assert len(set(pool["last_update"])) >= 2
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=len(pool) + 5000)
    ctx.pool_upload(pool)
    want_local, want_out = pyoracle.retire(pool, 1)
    got_out = ctx.pool_retire(1)
    assert len(want_out) > 0 and got_out.tobytes() == want_out.tobytes()
    assert ctx.pool_download().tobytes() == want_local.tobytes()
    ctx.pool_append(got_out[:100])
    after = ctx.pool_download()
    assert len(after) == len(pool) + 100 and after[len(pool):].tobytes() == got_out[:100].tobytes()
    ctx.close()


def test_pool_retire_with_a_too_small_buffer_leaves_the_pool_untouched():
    """dsm_pool_retire counts first: when the retired surfels do not fit the caller's buffer nothing is flagged dead,
    the call fails with DSM_E_CAPACITY and reports the needed size."""
    import ctypes
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    pose = synth.pose_stream(0)
    gray, depth = synth.make_frame(cam, 510, pose)
    _, pool = oracle_for(cam).fuse(4, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    assert len(pool) > 10
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=len(pool) + 64)
    ctx.pool_upload(pool)
    out, n = np.zeros(4, SURFEL_DTYPE), ctypes.c_int(0)
    rc = ctx.lib.dsm_pool_retire(ctx.h, 4, out.ctypes.data, 4, ctypes.byref(n))
    assert rc == -6 and n.value == len(pool)            # DSM_E_CAPACITY, *n_out = what a second call needs
    assert ctx.pool_download().tobytes() == pool.tobytes()  # nothing was retired
    assert ctx.pool_retire(4).tobytes() == pool.tobytes()   # with room: all of them, in pool order
    assert (ctx.pool_download()["update_times"] == 0).all()
    ctx.close()


def test_host_pointer_calls_invalidate_the_resident_pool():
    """dsm_fuse_frame / dsm_fuse_batch copy the caller's surfels into the buffer that holds the resident pool: afterwards the
    resident entry points must refuse (DSM_E_STATE) instead of running on overwritten data."""
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    pose = synth.pose_stream(0)
    gray, depth = synth.make_frame(cam, 511, pose)
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=1 << 16)
    # every pool call, each with its own cap so that none reaches the library through dsm_pool_size
    pool_calls = (ctx.pool_size, ctx.pool_download, lambda: ctx.fuse_frame_resident(1, gray, depth, pose),
                  lambda: ctx.pool_retire(0, cap=4), lambda: ctx.pool_export_cloud(1, cap=4),
                  lambda: ctx.pool_export_surfels(1, cap=4), lambda: ctx.pool_append(np.zeros(1, SURFEL_DTYPE)),
                  lambda: ctx.pool_transform(np.eye(4, dtype=np.float32)))

    def refused(calls):
        for call in calls:
            with pytest.raises(capi.DsmError) as e:
                call()
            assert e.value.code == -7  # DSM_E_STATE

    refused(pool_calls)  # before the first dsm_pool_upload
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.fuse_frame_resident(0, gray, depth, pose)
    assert ctx.pool_size() > 0
    _, new = ctx.fuse_frame(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))   # host-pointer call on the same context
    assert len(new) > 0
    refused(pool_calls)
    ctx.pool_upload(new)           # a fresh upload makes the resident mode usable again
    assert ctx.pool_size() == len(new)
    ctx.close()


@pytest.mark.parametrize("chunk", [1, 3, 4])
def test_stream_chunks_equal_frame_by_frame(chunk):
    """dsm_fuse_stream_resident (n frames per call) must leave exactly the pool that n calls of
    dsm_fuse_frame_resident leave: same kernels, same order on the pool, only batched differently."""
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    T = 8
    frames = []
    for t in range(T):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 600 + t, pose)
        frames.append((t // 2, gray, depth, pose))
    a = capi.Context(cam, max_batch=2, max_local_surfels=100000)
    a.pool_upload(np.zeros(0, SURFEL_DTYPE))
    counts_a = [a.fuse_frame_resident(r, g, d, p, want_count=True) for r, g, d, p in frames]
    want = a.pool_download()
    a.close()
    b = capi.Context(cam, max_batch=8, max_local_surfels=100000)
    b.pool_upload(np.zeros(0, SURFEL_DTYPE))
    counts_b = []
    for i in range(0, T, chunk):
        part = frames[i:i + chunk]
        c = b.fuse_stream_resident([f[0] for f in part], np.stack([f[1] for f in part]), np.stack([f[2] for f in part]),
                                   np.stack([f[3] for f in part]), want_counts=True)
        counts_b += list(c)
    got = b.pool_download()
    assert counts_b == counts_a
    assert got.tobytes() == want.tobytes()
    # mixing the two entry points on one context keeps working
    r, g, d, p = frames[0]
    b.fuse_frame_resident(9, g, d, p)
    b.fuse_stream_resident([9, 9], np.stack([g, g]), np.stack([d, d]), np.stack([p, p]))
    assert b.pool_size() > 0
    b.close()


@pytest.mark.parametrize("max_batch", [1, 2, 8])
def test_frame_resident_padded_rows_equal_packed_rows(max_batch):
    """dsm_fuse_frame_resident with padded rows (gray rows of W+24 bytes, depth rows of W+8 floats, the padding holding
    values no frame has), for gray, depth or both, must leave the pool byte-identical to the same stream with packed rows,
    with the same counts.  The C function is called directly: Context.fuse_frame_resident makes its inputs contiguous."""
    import ctypes
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    W, H = cam.width, cam.height
    frames = []
    for t in range(5):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 700 + t, pose)
        frames.append((t // 2, gray, depth, capi.pose16(pose)))
    pools, counts = [], []
    for padded in ((), ("gray",), ("depth",), ("gray", "depth")):
        ctx = capi.Context(cam, max_batch=max_batch, max_local_surfels=100000)
        ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
        cnt = []
        for ref, gray, depth, pose in frames:
            g, d = np.ascontiguousarray(gray), np.ascontiguousarray(depth)
            if "gray" in padded:
                g = np.full((H, W + 24), 255, np.uint8)
                g[:, :W] = gray
            if "depth" in padded:
                d = np.full((H, W + 8), 7.5, np.float32)
                d[:, :W] = depth
            n = ctypes.c_int(0)
            ctx._ck(ctx.lib.dsm_fuse_frame_resident(ctx.h, ref, g.ctypes.data, g.strides[0], d.ctypes.data, d.strides[0],
                                                    pose.ctypes.data, ctypes.byref(n)))
            cnt.append(n.value)
        pools.append(ctx.pool_download().tobytes())
        counts.append(cnt)
        ctx.close()
    assert min(counts[0]) > 0
    for k in range(1, len(pools)):
        assert counts[k] == counts[0], f"padded variant {k}"
        assert pools[k] == pools[0], f"padded variant {k}"


def test_inactive_store_round_trip():
    """Device-resident attached_surfels: retire two keyframes into the store, warp one of them, publish the inactive
    cloud, bring one back -- against the restated (and reference-pinned, tests/test_refmap.py) SurfelMap members."""
    import ctypes
    from densesurfelmapping_b200 import capi
    cam = synth.VGA
    orc = oracle_for(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    for t in range(3):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 500 + t, pose)
        lo, no = orc.fuse(t, gray, depth, pose, pool)
        pool = pyoracle.fuse_map_poststep(lo, no)
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=len(pool) + 5000)
    ctx.pool_upload(pool)
    store_calls = (lambda: ctx.inactive_retire(1), lambda: ctx.inactive_reactivate(1),
                   lambda: ctx.inactive_transform(1, np.eye(4, dtype=np.float32)), ctx.inactive_download,
                   ctx.inactive_export_cloud, lambda: ctx.inactive_export_poses([1]))

    def no_store():
        assert ctx.inactive_size() == (0, 0)
        for call in store_calls:
            with pytest.raises(capi.DsmError) as e:
                call()
            assert e.value.code == -7  # DSM_E_STATE

    no_store()
    ctx.inactive_reserve(16)
    with pytest.raises(capi.DsmError) as e:
        ctx.inactive_reserve(2 ** 31 - 1)  # 94 GB of surfels: more than the device holds
    assert e.value.code == -5  # DSM_E_NOMEM, and the store reserved before is gone
    no_store()
    ctx.inactive_reserve(3 * len(pool))
    loc1, out1 = pyoracle.retire(pool, 1)
    loc0, out0 = pyoracle.retire(loc1, 0)
    assert len(out1) > 0 and len(out0) > 0
    assert ctx.inactive_retire(1) == len(out1) and ctx.inactive_retire(0) == len(out0)
    assert ctx.inactive_retire(77) == 0
    assert ctx.inactive_size() == (len(out1) + len(out0), 2)
    assert ctx.pool_download().tobytes() == loc0.tobytes()
    assert ctx.inactive_download(1).tobytes() == out1.tobytes() and ctx.inactive_download(0).tobytes() == out0.tobytes()
    assert ctx.inactive_download().tobytes() == np.concatenate([out1, out0]).tobytes()
    # a cap below the count: the first cap surfels are written, nothing past them, and *n_out is the full count
    for kf, want in ((-1, np.concatenate([out1, out0])), (0, out0)):
        cap = len(want) - len(out0) // 2
        buf = np.frombuffer(b"\xab" * (len(want) * SURFEL_DTYPE.itemsize), SURFEL_DTYPE).copy()
        n = ctypes.c_int(0)
        assert ctx.lib.dsm_inactive_download(ctx.h, kf, buf.ctypes.data, cap, ctypes.byref(n)) == 0
        assert n.value == len(want) and buf[:cap].tobytes() == want[:cap].tobytes()
        assert buf[cap:].tobytes() == b"\xab" * ((len(want) - cap) * SURFEL_DTYPE.itemsize)
    a = np.deg2rad(2.0)
    Wm = np.eye(4)
    Wm[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    Wm[:3, 3] = [0.5, -0.1, 0.25]
    w = np.ascontiguousarray(Wm.T.astype(np.float32).reshape(16))
    ctx.inactive_transform(1, w)
    warped1 = pyoracle.warp_active(out1, w)
    check_surfels(ctx.inactive_download(1), warped1, "warped segment")
    assert ctx.inactive_download(0).tobytes() == out0.tobytes()            # the other pose did not move
    store = ctx.inactive_download()
    pts = ctx.inactive_export_cloud()
    assert pts.tobytes() == pyoracle.cloud_points(store, -(2 ** 31)).tobytes()
    seg1 = ctx.inactive_download(1)
    assert ctx.inactive_reactivate(1) == len(out1)
    assert ctx.inactive_size() == (len(out0), 1)
    assert ctx.inactive_download().tobytes() == out0.tobytes()             # the gap was closed
    after = ctx.pool_download()
    assert len(after) == len(loc0) + len(seg1) and after[len(loc0):].tobytes() == seg1.tobytes()
    ctx.close()


def test_inactive_capacity_errors_change_nothing():
    """dsm_inactive_retire fails with DSM_E_CAPACITY when the store size plus the exact pool size exceeds the
    reservation, dsm_inactive_reactivate when the pool size plus the keyframe's stored surfels exceeds max_local_surfels.
    A rejected call leaves the pool, the store and both exports byte-identical, and the next call that fits succeeds."""
    from densesurfelmapping_b200 import capi
    rng = np.random.default_rng(11)
    pool = np.zeros(300, SURFEL_DTYPE)
    for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
        pool[f] = rng.standard_normal(len(pool))
    pool["update_times"] = 3
    pool["last_update"] = np.arange(len(pool)) % 3  # 100 surfels each of keyframes 0, 1, 2, interleaved

    def state(ctx):
        return (ctx.pool_download().tobytes(), ctx.inactive_download().tobytes(), ctx.inactive_size(),
                ctx.inactive_export_cloud().tobytes(), ctx.inactive_export_poses([0, 1, 2]).tobytes())

    def rejected(ctx, call, kf):
        before = state(ctx)
        with pytest.raises(capi.DsmError) as e:
            call(kf)
        assert e.value.code == -6
        assert state(ctx) == before

    def new_ctx(cap, store):
        ctx = capi.Context(synth.VGA, max_batch=2, max_local_surfels=cap)
        ctx.pool_upload(pool)
        ctx.inactive_reserve(store)
        assert ctx.inactive_retire(1) == 100
        return ctx

    ctx = new_ctx(400, 350)
    rejected(ctx, ctx.inactive_retire, 0)          # 100 stored + 300 in the pool > 350
    assert ctx.inactive_reactivate(1) == 100       # 300 + 100 <= 400
    assert ctx.inactive_size() == (0, 0) and ctx.pool_size() == 400
    ctx.close()
    ctx = new_ctx(399, 400)
    rejected(ctx, ctx.inactive_reactivate, 1)      # 300 in the pool + 100 stored > 399
    assert ctx.inactive_retire(0) == 100           # 100 + 300 <= 400
    assert ctx.inactive_size() == (200, 2)
    assert ctx.inactive_download().tobytes() == np.concatenate([pool[pool["last_update"] == k] for k in (1, 0)]).tobytes()
    ctx.close()
