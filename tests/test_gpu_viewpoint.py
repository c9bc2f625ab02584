"""dsm_viewpoint_enable / _enqueue / _wait: clear candidate positions around each frontier cluster, each scored at its
best rotation by the sampled cluster voxels it would see through the latest known field.

The device equals oracle/pyoracle_viewpoint bit for bit in the header and every record: on every known field of the
windowed drive (chunks 1 and 4, warps between calls, three shapes and voxel edges, with and without reach, both
blocking rules, 8- and 64-rotation tables with pitched entries; the model runs on the device's own field_state and
distances), with a resident twin of each request; on grids loaded through dsm_debug_field_load_state (hand cases, a
64x48x24 density sweep, 320x320x40 at 128 voxels of range, a sampling cut).  Each returned viewpoint, re-scored by a gain
job at its pose naming its cluster, gives n_cluster == n_seen; with reach each cost is the host-copy reach cost grid's.
Stream order, a drive beside publish snapshots and asynchronous checkpoints against a twin without viewpoint jobs, the
rejected frame and every error code are checked too.  The node is checked through tests/cpp/viewpoint_main.cpp."""
import ctypes
from functools import partial

import numpy as np
import pytest

import known_space
import pyoracle_frontier
import pyoracle_gain as G
import pyoracle_reach
import pyoracle_viewpoint as V
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, NODE_FIELD, assert_error_stays, gcam, known_drive,
                         node_args, rejected, rejected_known, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import open_room, params, rotations, scene
from resident_map import SHAPES, camera, load_known

pytestmark = pytest.mark.gpu

INF = V.INF
ROT8 = np.concatenate([rotations(4), rotations(2, (0.35, -0.35))])
ROT64 = rotations(16, (0.0, 0.3, -0.3, 0.6))


same = partial(known_space.same, names=("header", "clusters", "viewpoints"))


def loader(shape, voxel=0.2, max_clusters=64, max_candidates=1 << 16, reach=False, gain=0):
    ctx = small_ctx(shape, voxel)
    ctx.frontier_enable(256, 1 << 18)
    if reach:
        ctx.reach_enable(16, 1 << 12, 4096)
    if gain:
        ctx.gain_enable(gain)
    ctx.viewpoint_enable(max_clusters, max_candidates)
    return ctx


def rescore(ctx, got, frontier, cam, rot, origin, voxel, shape_zyx):
    """Every returned viewpoint of a cluster whose members are all samples, scored by a gain job at its pose naming its
    cluster: n_cluster == n_seen."""
    _, recs, slots = got
    poses, cl, want = [], [], []
    nz, ny, nx = shape_zyx
    for i, r in enumerate(recs):
        if r["status"] != 0 or r["n_samples"] != frontier[0][r["cluster"]]["n_voxels"]:
            continue
        for s in slots[i]:
            if s["voxel"] < 0:
                continue
            c = np.array([s["voxel"] % nx, s["voxel"] // nx % ny, s["voxel"] // (nx * ny)])
            t = G.centres([c], origin, voxel)[0]
            poses.append(np.concatenate([rot[s["rotation"]].reshape(3, 3), t[:, None]], axis=1).reshape(12))
            cl.append(r["cluster"])
            want.append(s["n_seen"])
    if not poses:
        return 0
    ctx.gain_enqueue(cam, poses, np.array(cl, np.int32))
    _, g = ctx.gain_wait()
    assert g["n_cluster"].tolist() == want
    return len(poses)


def loaded(ctx, state, origin, voxel, cam, rot, prm, clusters=None, m=1, what="", reach_start=None):
    """Loads the grid, runs a frontier job (and a reach job from reach_start with host_copy) and the viewpoint job
    against the model on the same grids."""
    dist = load_known(ctx, state, origin, voxel, what)
    ctx.frontier_enqueue(m)
    fc, fv, _ = ctx.frontier_wait()
    cost = None
    if reach_start is not None:
        ctx.reach_enqueue(reach_start, prm.radius, 1, None, False, True)
        cost = ctx.reach_wait()[3]
    cl = np.arange(min(len(fc), 24)) if clusters is None else clusters
    ctx.viewpoint_enqueue(cam, rot, cl, prm)
    got = ctx.viewpoint_wait()
    same(got, V.viewpoints(state, dist, origin, voxel, cam, rot, cl, prm, (fc, fv), cost), what)
    return got, (fc, fv), cost


def test_hand_cases():
    voxel = 0.25
    st = open_room()
    ctx = loader(st.shape[::-1], voxel, reach=True, gain=256)
    for ub in (0, 1):
        for rot in (ROT8, ROT64):
            cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 3.0, ub)
            prm = params(0, 6, 1, 1, top_k=16)
            got, fr, _ = loaded(ctx, st, (0, 0, 0), voxel, cam, rot, prm, [0, 1, 5], what=f"room ub={ub}")
            assert got[1]["status"].tolist() == [0, 3, 3] and got[1][0]["n_viewpoints"] == 16
            assert rescore(ctx, got, fr, cam, rot, (0, 0, 0), voxel, st.shape) == 16
            got, _, cost = loaded(ctx, st, (0, 0, 0), voxel, cam, rot, prm._replace(with_reach=1, radius=0.3), [0],
                                  what=f"room reach ub={ub}", reach_start=G.centres([(3, 3, 1)], (0, 0, 0), voxel)[0])
            s = got[2][0][got[2][0]["voxel"] >= 0]
            assert (s["cost"] == cost.reshape(-1)[s["voxel"]]).all() and (s["cost"] != INF).all()
    # a sealed pocket: traversable candidates that the reach job does not reach
    st = np.full((3, 13, 13), FREE, np.uint8)
    st[:, 12, :] = UNKNOWN
    st[:, 4:10, 0:5] = OCCUPIED
    st[:, 5:9, 1:4] = FREE
    ctx.close()
    ctx = loader(st.shape[::-1], voxel, reach=True)
    cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 3.0, 1)
    got, _, _ = loaded(ctx, st, (0, 0, 0), voxel, cam, ROT8, params(0, 6, 1, 1, top_k=16, with_reach=1), [0], what="pocket",
                       reach_start=G.centres([(10, 2, 1)], (0, 0, 0), voxel)[0])
    assert 0 < got[1][0]["n_reached"] < got[1][0]["n_traversable"]
    ctx.close()


def test_random_grids_over_a_density_sweep():
    shape, voxel, o = (64, 48, 24), 0.2, (-30, -20, -4)
    ctx = loader(shape, voxel, reach=True, gain=1024)
    rng = np.random.default_rng(21)
    for n_blobs, p_occ in [(4, 0.02), (12, 0.05), (30, 0.1), (60, 0.02), (120, 0.15)]:
        st = scene(rng, shape, n_blobs, p_occ)
        start = G.centres([(32, 24, 12)], o, voxel)[0]
        x, y, z = 32, 24, 12
        st[z, y, x] = FREE
        for ub, R, rot, prm in [(1, 8 * voxel, ROT8, params(1, 4, 1, 1, top_k=4)),
                                (0, 20 * voxel, ROT64, params(2, 8, 2, 2, top_k=8, max_samples=64, min_seen=2)),
                                (1, 12 * voxel, ROT64, params(0, 6, 0, 3, top_k=16, with_reach=1, radius=0.1))]:
            cam = gcam(K, R, ub)
            got, fr, _ = loaded(ctx, st, o, voxel, cam, rot, prm, m=1 + ub, what=f"blobs {n_blobs} ub={ub}",
                                reach_start=start if prm.with_reach else None)
            if prm.max_samples >= 4096:
                rescore(ctx, got, fr, cam, rot, o, voxel, st.shape)
    ctx.close()


def test_a_size_a_user_runs_at_the_longest_range():
    shape, voxel, o = (320, 320, 40), 0.2, (-160, -160, -5)
    rng = np.random.default_rng(6)
    st = scene(rng, shape, 40, 0.01)
    ctx = loader(shape, voxel, max_candidates=1 << 20)
    cam = gcam(SMALL_CAM, 128 * voxel, 1)
    got, _, _ = loaded(ctx, st, o, voxel, cam, ROT8, params(4, 12, 2, 4, top_k=4, max_samples=256), np.arange(6),
                       what="320x320x40 at 128 v")
    assert (got[1]["n_viewpoints"] > 0).sum() >= 1
    ctx.close()


def test_sampling_cut():
    shape, voxel = (40, 36, 8), 0.2
    st = np.full(shape[::-1], FREE, np.uint8)
    st[:, 30:, :] = UNKNOWN                   # one frontier wall of 40 x 8 voxels
    ctx = loader(shape, voxel)
    cam = G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 4.0, 1)
    for ms in (1, 7, 100, 320, 4096):
        got, _, _ = loaded(ctx, st, (0, 0, 0), voxel, cam, ROT8, params(2, 10, 2, 2, top_k=6, max_samples=ms), [0], what=f"cut {ms}")
        assert got[1][0]["n_samples"] == min(ms, 320)
    ctx.close()


def test_stream_order():
    """A job reads the field, frontier and reach results it was enqueued behind, not the next field request, frontier
    job or reach job; it needs a frontier job, and with reach a reach job, on the latest field request."""
    shape, voxel = (40, 30, 12), 0.2
    ctx = loader(shape, voxel, reach=True)
    rng = np.random.default_rng(9)
    a, b = scene(rng, shape, 10), scene(rng, shape, 25)
    start = G.centres([(20, 15, 6)], (0, 0, 0), voxel)[0]
    a[6, 15, 20] = b[6, 15, 20] = FREE
    cam = gcam(K, 10 * voxel, 1)
    prm = params(1, 5, 1, 1, top_k=4, with_reach=1)
    cl = np.arange(6)
    ctx.debug_field_load_state(a, (0, 0, 0))
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue(cam, ROT8, cl, prm)            # no frontier job on this field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue(cam, ROT8, cl, prm)            # with reach, no reach job on this field
    assert e.value.code == -7
    ctx.reach_enqueue(start, 0.0, 1, None, False, True)
    ctx.viewpoint_enqueue(cam, ROT8, cl, prm)                # before the field is waited for
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue(cam, ROT8, cl, prm)            # one job in flight
    assert e.value.code == -7
    fa = ctx.field_wait()
    ra = ctx.reach_wait()
    fra = ctx.frontier_wait()
    got = ctx.viewpoint_wait()
    want = V.viewpoints(a, fa[0], (0, 0, 0), voxel, cam, ROT8, cl, prm, fra[:2], ra[3])
    same(got, want, "first")
    ctx.frontier_enqueue(1)
    ctx.reach_enqueue(start, 0.0, 1, None, False, False)
    ctx.viewpoint_enqueue(cam, ROT8, cl, prm)
    ctx.debug_field_load_state(b, (5, 5, 5))                 # the next field request, while the job is in flight
    ctx.frontier_wait()
    ctx.frontier_enqueue(1)                                  # the next frontier and reach jobs
    ctx.reach_wait()
    ctx.reach_enqueue(start + 1.0, 0.0, 1, None, False, False)
    got = ctx.viewpoint_wait()
    ctx.field_wait()
    ctx.frontier_wait()
    ctx.reach_wait()
    same(got, want, "the old field, frontiers and costs")
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    ctx.viewpoint_enqueue(cam, ROT8, cl, prm._replace(with_reach=0))
    ctx.viewpoint_wait()
    ctx.field_enqueue((0, 0, 0), 1)                          # a plain request
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue(cam, ROT8, cl, prm._replace(with_reach=0))
    assert e.value.code == -7
    ctx.field_wait()
    ctx.close()


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_fields_of_the_drive(chunk, shape):
    """The windowed drive with loop-closure warps between calls; after every call a known field, its frontiers, a reach
    job from the camera with its host copy, and a viewpoint job over the clusters, against the model on the field's
    own grids; the viewpoints re-scored by gain jobs; the same job on a resident twin of the request equals it."""
    def enable(c):
        c.frontier_enable(64, 1 << 16)
        c.reach_enable(16, 1 << 12, 2048)
        c.gain_enable(2048)
        c.viewpoint_enable(64, 1 << 18)

    found = 0
    for call, t0, t1, ctx, v, cam, slots, poses, (dist, origin, _), state in known_drive(shape, chunk, (0.125, 0.1, 0.3), enable):
        ctx.frontier_enqueue(1 + call % 3)
        fc, fv, _ = ctx.frontier_wait()
        with_reach = call % 2
        ctx.reach_enqueue(cam, 0.0, 1, None, False, True)
        cost = ctx.reach_wait()[3]
        ub = (call // 2) % 2
        rot = ROT64 if call % 3 == 2 else ROT8
        gc = gcam(K, (10 + 7 * (call % 3)) * np.float32(v), ub)
        prm = params(1 + call % 2, 4, 1, 1 + call % 3, top_k=1 + 5 * (call % 4), with_reach=with_reach,
                     radius=0.05 * (call % 2))
        cl = (np.arange(min(len(fc) + 2, 12)) if len(fc) else np.array([0, 3])).astype(np.int32)
        ctx.viewpoint_enqueue(gc, rot, cl, prm)
        got = ctx.viewpoint_wait()
        what = f"frames {t0}-{t1 - 1}, voxel {v}"
        same(got, V.viewpoints(state, dist, origin, v, gc, rot, cl, prm, (fc, fv), cost if with_reach else None), what)
        rescore(ctx, got, (fc, fv), gc, rot, origin, v, state.shape)
        found += int(got[1]["n_viewpoints"].sum())
        if with_reach:
            s = got[2][got[2]["voxel"] >= 0]
            assert (s["cost"] == cost.reshape(-1)[s["voxel"]]).all(), what
        # a resident twin of the same request
        ctx.field_enqueue_known(cam, 5, slots, poses, host_copy=False)
        ctx.field_wait()
        ctx.frontier_enqueue(1 + call % 3)
        ctx.frontier_wait()
        ctx.reach_enqueue(cam, 0.0, 1, None, False, False)
        ctx.reach_wait()
        ctx.viewpoint_enqueue(gc, rot, cl, prm)
        twin = ctx.viewpoint_wait()
        assert all(a.tobytes() == b.tobytes() for a, b in zip(twin, got)), f"{what}: resident twin"
    assert found > 0 or shape == (1, 1, 1)


def test_viewpoint_jobs_change_nothing_else(tmp_path):
    """A drive with frontier, reach and viewpoint jobs beside a publish snapshot and an asynchronous checkpoint leaves
    the map, both published clouds, the fields, the state grids, the frontiers, the reach results and the checkpoint
    files byte-identical to a twin without viewpoint jobs."""
    prm = params(1, 5, 1, 1, top_k=3, with_reach=1)

    def enable_both(c):
        c.frontier_enable(32, 4096)
        c.reach_enable(16, 1 << 12, 1024)

    def enqueue(c, is_a, call, t1):
        c.frontier_enqueue(1)
        c.reach_enqueue(camera(t1 - 1), 0.1, 2, [camera(0)], True, True)
        if is_a:
            c.viewpoint_enqueue(gcam(K, 20 * 0.1, call % 2), ROT8, np.arange(8), prm)

    def check(a, outs, call, t1, what):
        want = V.viewpoints(outs["state"][0], outs["field"][0], outs["field"][1], 0.1, gcam(K, 20 * 0.1, call % 2), ROT8, np.arange(8),
                            prm, outs["shared"]["frontiers"][:2], outs["shared"]["reach"][3])
        same(a.viewpoint_wait(), want, what)

    twin_drive(tmp_path, enable_both, lambda a: a.viewpoint_enable(32, 1 << 16), enqueue,
               lambda c: {"frontiers": c.frontier_wait(), "reach": c.reach_wait()}, check)


def test_rejected_frame_comes_back_from_wait():
    gc, prm = gcam(K, 30 * 0.1, 0), params(1, 6, 1, 1, top_k=2)

    def enable(b):
        b.frontier_enable(32, 1 << 14)
        b.viewpoint_enable(32, 1 << 16)

    def enqueue(b, first):
        b.frontier_enqueue(1)
        b.viewpoint_enqueue(gc, ROT8, np.arange(8), prm)

    r = rejected_known(enable, enqueue)
    dist, origin, _ = r.field
    fr = rejected(r.ctx.frontier_wait).frontier
    e = rejected(r.ctx.viewpoint_wait)
    same(e.viewpoint, V.viewpoints(r.state, dist, origin, r.voxel, gc, ROT8, np.arange(8), prm, fr[:2]), "rejected")
    assert e.viewpoint[1]["n_traversable"].sum() > 0
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    st = open_room()
    ok = capi.DsmGainCamera(4.0, 4.0, 3.5, 3.5, 8, 8, 2.0, 1)
    rot = np.ascontiguousarray(ROT8)
    R = rot.ctypes.data
    cl = np.zeros(1, np.int32)
    C = cl.ctypes.data

    def prm(**kw):
        p = capi.DsmViewpointParams(1, 3, 1, 1, 4096, 0, 4, 0, 0.0, 0)
        for k, v in kw.items():
            setattr(p, k, v)
        return ctypes.byref(p)

    def enq(cam=ctypes.byref(ok), r=R, n_rot=8, c=C, n=1, p="default"):
        return lib.dsm_viewpoint_enqueue(ctx.h, cam, r, n_rot, c, n, prm() if p == "default" else p)

    assert lib.dsm_viewpoint_enable(ctx.h, 1, 1) == -7                  # before dsm_field_enable
    ctx.field_enable(0.25, 12, 13, 3)
    assert lib.dsm_viewpoint_enable(ctx.h, 1, 1) == -7                  # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert enq() == -7                                                  # before dsm_viewpoint_enable
    assert lib.dsm_viewpoint_wait(ctx.h, None, None, None) == -7
    for a, b in [(0, 1), (4097, 1), (1, 0), (1, (1 << 22) + 1), (-1, 1)]:
        assert lib.dsm_viewpoint_enable(ctx.h, a, b) == -1, (a, b)
    assert lib.dsm_viewpoint_enable(None, 1, 1) == -1
    ctx.viewpoint_enable(4, 200)
    assert lib.dsm_viewpoint_enable(ctx.h, 1, 1) == -7                  # once
    assert enq() == -7                                                  # no field request yet
    assert lib.dsm_viewpoint_wait(ctx.h, None, None, None) == -7        # nothing enqueued
    ctx.field_enqueue((0, 0, 0), 1)                                     # a plain request
    ctx.field_wait()
    assert enq() == -7
    load_known(ctx, st, (0, 0, 0), 0.25)
    assert enq() == -7                                                  # no frontier job on this field
    ctx.frontier_enable(8, 1024)
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    assert enq(p=prm(with_reach=1)) == -7                               # no reach job
    ctx.reach_enable(4, 64, 64)
    ctx.reach_enqueue((0.6, 0.6, 0.4), 0.0, 1)
    ctx.reach_wait()
    load_known(ctx, st, (0, 0, 0), 0.25)
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    assert enq(p=prm(with_reach=1)) == -7                               # the reach job read the old field
    nan, inf = float("nan"), float("inf")
    bad = []
    for field, value in [("fx", 0.0), ("fy", nan), ("cx", inf), ("width", 0), ("height", 65537), ("max_range", 0.0),
                         ("max_range", 32.1), ("max_range", nan), ("unknown_blocks", 2)]:
        c = capi.DsmGainCamera(4.0, 4.0, 3.5, 3.5, 8, 8, 2.0, 1)
        setattr(c, field, value)
        bad.append(dict(cam=ctypes.byref(c)))
    r2 = rot.copy()
    r2[3, 4] = nan
    cl2 = np.array([-1], np.int32)
    bad += [dict(cam=None), dict(r=None), dict(n_rot=0), dict(n_rot=65), dict(r=r2.ctypes.data), dict(c=None), dict(n=-1), dict(n=5),
            dict(c=cl2.ctypes.data), dict(p=None)]
    for kw in [dict(r_min=-1), dict(r_min=4), dict(r_max=65), dict(dz_max=-1), dict(dz_max=17), dict(stride=0), dict(stride=9),
               dict(max_samples=0), dict(max_samples=4097), dict(min_seen=-1), dict(top_k=0), dict(top_k=17), dict(with_reach=2),
               dict(radius=nan), dict(radius=-0.5), dict(radius=inf), dict(r_min=3, r_max=3, stride=2)]:
        bad.append(dict(p=prm(**kw)))
    two = np.zeros(2, np.int32)
    bad.append(dict(p=prm(r_max=4), n=2, c=two.ctypes.data))           # 2 x 144 candidates above 200
    bad.append(dict(p=prm(r_min=0, r_max=19, dz_max=1)))                # 3 layers of 1 257 offsets above 4096
    for kw in bad:
        assert enq(**kw) == -1, kw
    assert lib.dsm_viewpoint_enqueue(None, ctypes.byref(ok), R, 8, C, 1, prm()) == -1
    assert enq(p=prm(r_max=4)) == 0                                     # 144 candidates pass
    assert enq() == -7                                                  # one job in flight
    info = np.zeros(1, capi.VIEWPOINT_INFO_DTYPE)
    assert lib.dsm_viewpoint_wait(ctx.h, info.ctypes.data, None, None) == 0
    assert info[0]["n_clusters"] == 1 and info[0]["reserved"].tolist() == [0] * 6
    assert lib.dsm_viewpoint_wait(ctx.h, None, None, None) == -7
    assert enq(c=None, n=0) == 0                                        # no clusters
    info, recs, slots = ctx.viewpoint_wait()
    assert info["n_clusters"] == 0 and len(recs) == 0 and slots.shape == (0, 4)
    ctx.close()
    # the work bound: n_clusters n_offsets max_samples <= 2^31
    ctx = loader((12, 13, 3), 0.25, max_clusters=4096, max_candidates=1 << 22)
    load_known(ctx, st, (0, 0, 0), 0.25)
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    n_off = len(V.offsets(params(0, 6, 1, 1)))
    k = V.MAX_WORK // (n_off * 4096)
    assert k * n_off <= V.MAX_CANDIDATES and k < V.MAX_CLUSTERS
    big = capi.DsmViewpointParams(0, 6, 1, 1, 4096, 0, 1, 0, 0.0, 0)
    many = np.zeros(k + 1, np.int32)
    assert lib.dsm_viewpoint_enqueue(ctx.h, ctypes.byref(ok), R, 8, many.ctypes.data, k + 1, ctypes.byref(big)) == -1
    assert lib.dsm_viewpoint_enqueue(ctx.h, ctypes.byref(ok), R, 8, many.ctypes.data, k, ctypes.byref(big)) == 0
    info, recs, _ = ctx.viewpoint_wait()
    assert info["n_clusters"] == k and (recs["status"] == 0).all()
    assert len(set(recs[["n_samples", "n_inside", "n_traversable", "n_viewpoints"]].tolist())) == 1
    ctx.close()


# ---- the node ----
def test_node_viewpoints_equal_the_model_and_change_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers(), reach() and viewpoints() over
    every cluster, with reach on every other frame, equal the model over the grids, frontiers, reach start and rotations
    the driver dumps (the reach job's costs being Dijkstra's from its start); clouds,
    PLY and PCD files equal a twin without viewpoint jobs; viewpoints() after load_state until the next fused frame
    returns DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("viewpoint_main", str(tmp_path), cam, sc, node_args() + [1, RELOAD], tag="a", after=[pa])
    q = run_driver("viewpoint_main", str(tmp_path), cam, sc, node_args() + [0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, ub = r.i(), r.i()
        max_range = float(r.take(np.float32, 1)[0])
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        rinfo = r.take(np.uint8, pyoracle_reach.INFO_DTYPE.itemsize).view(pyoracle_reach.INFO_DTYPE)[0].copy()
        rot = r.lst(np.float64).reshape(-1, 9)
        named = r.lst(np.int32)
        prm = V.Params(*r.take(np.int32, 8).tolist(), float(r.take(np.float32, 1)[0]))
        info = r.take(np.uint8, V.INFO_DTYPE.itemsize).view(V.INFO_DTYPE)[0].copy()
        recs = r.lst(V.CLUSTER_DTYPE)
        slots = r.lst(V.VIEWPOINT_DTYPE).reshape(len(recs), -1)
        after_load = r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        gc = G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, max_range, ub)
        cost = None
        if prm.with_reach:     # the reach job from the middle voxel converged, so its costs are Dijkstra's
            assert rinfo["converged"] == 1, f"message {t}"
            cost = pyoracle_reach.dijkstra(pyoracle_reach.traversable(state, dist, prm.radius), int(rinfo["start_voxel"]))
        want = V.viewpoints(state, dist, origin, voxel, gc, rot, named, prm, (clusters, vox), cost)
        same((info, recs, slots), want, f"message {t}")
        found += int((recs["n_viewpoints"] > 0).sum()) > 0
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: viewpoints() after load_state"
    assert found > 0
    twin_node_tail(r, q, pa, pb)
