"""dsm_gain_enable / _enqueue / _wait: the frustum, free, unknown, occupied, frontier and cluster voxels each candidate
camera pose would see through the latest known field.

The device equals oracle/pyoracle_gain bit for bit in every record and header: on every known field of the windowed
drive (views at eight yaws around each viewpoint of a reach job and random poses, both blocking rules, with and without
clusters; the model runs on the device's own field_state, which tests/test_gpu_field_known.py pins to the known-space
oracle); on grids loaded through dsm_debug_field_load_state (hand cases, a density sweep, 320x320x40 at the longest
range, a request of max_views views against the model on a subset and against smaller requests; each load's distances,
counts and states are held to the known-space oracle first, through resident_map.load_known); a resident field
against its host-copy twin; the stream order against the next field request and the next frontier job; a drive with gain
jobs beside publish snapshots and asynchronous checkpoints leaves everything as a twin without them; the rejected-frame
and error contracts.  The node is checked through tests/cpp/gain_main.cpp."""
import ctypes
import filecmp

import numpy as np
import pytest

import pyoracle_frontier
import pyoracle_gain as G
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import SHAPES, STORE, T, camera, load_known, map_state, new_ctx, simple_lists, warp, windowed
from test_gain_model import random_pose, symmetric_scene, symmetric_views, wall_scene, yaw_pose
from test_gpu_field_known import MAX_RANGE, Views

pytestmark = pytest.mark.gpu

SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
K = synth.KITTI
UNKNOWN, OCCUPIED, FREE = G.UNKNOWN, G.OCCUPIED, G.FREE


def gcam(cam, max_range, unknown_blocks):
    return G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, float(np.float32(max_range)), unknown_blocks)


def same(got, want, what):
    gi, gg = got
    wi, wg = want
    assert gi.tobytes() == np.array(wi).tobytes(), f"{what}: header {gi} want {wi}"
    bad = np.flatnonzero(gg != wg)
    assert gg.tobytes() == wg.tobytes(), f"{what}: {len(bad)} records differ, first {bad[:4]}\n{gg[bad[:4]]}\nwant\n{wg[bad[:4]]}"


def loader(shape, voxel=0.2, max_views=64, frontier_caps=(256, 1 << 18)):
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(*frontier_caps)
    ctx.gain_enable(max_views)
    return ctx


def job(ctx, state, origin, voxel, cam, poses, clusters=None, m=1):
    """The device's job on the latest (waited) known field against the model on its state grid."""
    fr = None
    if clusters is not None:
        ctx.frontier_enqueue(m)
        fc, fv, _ = ctx.frontier_wait()
        fr = (fc, fv)
    ctx.gain_enqueue(cam, poses, clusters)
    return ctx.gain_wait(), G.gains(state, origin, voxel, cam, poses, clusters, fr)


def loaded(ctx, state, origin, voxel, cam, poses, clusters=None, m=1, what=""):
    load_known(ctx, state, origin, voxel, what)
    got, want = job(ctx, state, origin, voxel, cam, poses, clusters, m)
    same(got, want, what)
    return got


def some_clusters(rng, n, n_views):
    return rng.integers(-1, n + 2, size=n_views).astype(np.int32)


def test_hand_cases():
    voxel = 0.5
    ctx = loader((12, 5, 5), voxel)
    c = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 5.5, 1)
    t = G.centres([(1, 2, 2)], (0, 0, 0), voxel)[0]
    poses = [yaw_pose(k, t) for k in range(4)] + [yaw_pose(0, t + 0.3), yaw_pose(0, G.centres([(-2, 2, 2)], (0, 0, 0), voxel)[0])]
    for kind in (OCCUPIED, UNKNOWN, FREE):
        for ub in (0, 1):
            got = loaded(ctx, wall_scene(kind), (0, 0, 0), voxel, c._replace(unknown_blocks=ub), poses, [0, 1, -1, 5, 0, 0],
                         what=f"wall {kind} ub={ub}")
            assert got[1]["status"][5] == 1
    ctx.close()
    # the image edges, voxels behind the camera and a centre at max_range, in exact arithmetic
    ctx = loader((5, 1, 5), 1.0)
    pose = np.concatenate([np.eye(3), np.array([[0.5], [0.5], [0.5]])], axis=1).reshape(12)
    for R in (2.0, 2.5, float(np.nextafter(np.float32(2.0), np.float32(0)))):
        got = loaded(ctx, np.full((5, 1, 5), FREE, np.uint8), (0, 0, 0), 1.0, G.Camera(1.0, 1.0, 0.0, 0.5, 1, 1, R, 1), [pose],
                     what=f"edges R={R}")
    assert got[1]["n_frustum"][0] == 1
    ctx.close()
    # a camera outside the grid, in an unknown voxel, in a corner (a clipped box), and axes of one voxel
    rng = np.random.default_rng(2)
    for shape, o, voxel in [((8, 7, 6), (3, 3, 3), 0.25), ((1, 1, 1), (0, 0, 0), 0.5), ((5, 1, 1), (-2, 0, 0), 0.5),
                            ((1, 6, 1), (0, 0, 0), 0.5), ((1, 1, 7), (0, 0, 9), 0.5)]:
        ctx = loader(shape, voxel)
        for p in [(0.1, 0.1, 0.8), (0.3, 0.0, 0.7)]:
            st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
            c0 = G.centres([(0, 0, 0)], o, voxel)[0]
            poses = [yaw_pose(k, c0 + 0.05) for k in range(4)] + [random_pose(rng, c0, 3 * voxel) for _ in range(8)]
            poses.append(yaw_pose(0, c0 - 3 * voxel))
            for ub in (0, 1):
                cam = G.Camera(3.0, 3.0, 2.0, 2.0, 4, 4, 4 * voxel, ub)
                loaded(ctx, st, o, voxel, cam, poses, some_clusters(rng, 3, len(poses)), what=f"{shape} {p} ub={ub}")
        ctx.close()
    # the yaw symmetry
    n, nz = 15, 7
    ctx = loader((n, n, nz), 0.5)
    st = symmetric_scene(n, nz, np.random.default_rng(17))
    _, poses = symmetric_views(n, nz, 0.5)
    for ub in (0, 1):
        got = loaded(ctx, st, (0, 0, 0), 0.5, G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 3.5, ub), poses, what=f"symmetry ub={ub}")
        assert all(got[1][k].tobytes() == got[1][0].tobytes() for k in range(4))
    ctx.close()


def test_random_grids_over_a_density_sweep():
    shape, voxel, o = (64, 48, 24), 0.2, (-30, -20, -4)
    ctx = loader(shape, voxel, max_views=96)
    rng = np.random.default_rng(21)
    for p in [(0.1, 0.1, 0.8), (0.2, 0.1, 0.7), (0.3, 0.1, 0.6), (0.05, 0.3, 0.65), (0.0, 0.5, 0.5)]:
        st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
        centre = G.centres([(32, 24, 12)], o, voxel)[0]
        poses = [random_pose(rng, centre, 5.0) for _ in range(40)]
        for ub, R in [(1, 8 * voxel), (0, 20 * voxel)]:
            cam = gcam(K, R, ub)
            loaded(ctx, st, o, voxel, cam, poses, some_clusters(rng, 30, len(poses)), m=1 + ub, what=f"density {p} ub={ub}")
            loaded(ctx, st, o, voxel, cam, poses, what=f"density {p} ub={ub}, no clusters")
    ctx.close()


def test_a_size_a_user_runs_at_the_longest_range():
    shape, voxel, o = (320, 320, 40), 0.2, (-160, -160, -5)
    rng = np.random.default_rng(6)
    st = rng.choice(3, size=shape[::-1], p=(0.02, 0.01, 0.97)).astype(np.uint8)
    ctx = loader(shape, voxel, max_views=8)
    centre = G.centres([(160, 160, 20)], o, voxel)[0]
    poses = [yaw_pose(0, centre), yaw_pose(3, centre + np.array([7.0, -3.0, 0.1]))]
    for p in poses:   # the cameras stand in free voxels
        x, y, z = (np.floor(p.reshape(3, 4)[:, 3] / np.float64(np.float32(voxel))) - o).astype(int)
        st[z, y, x] = FREE
    got = loaded(ctx, st, o, voxel, gcam(SMALL_CAM, 128 * voxel, 1), poses, what="320x320x40 at 128 v")
    assert (got[1]["n_free"] > 1000).all()
    ctx.close()


def test_the_most_views_one_request_takes():
    shape, voxel, o = (96, 80, 24), 0.2, (0, 0, 0)
    max_views = 1 << 14
    rng = np.random.default_rng(14)
    st = rng.choice(3, size=shape[::-1], p=(0.2, 0.05, 0.75)).astype(np.uint8)
    ctx = loader(shape, voxel, max_views=max_views)
    load_known(ctx, st, o, voxel)
    ctx.frontier_enqueue(1)
    fr = ctx.frontier_wait()[:2]
    centre = G.centres([(48, 40, 12)], o, voxel)[0]
    poses = np.stack([random_pose(rng, centre, 9.0) for _ in range(max_views)])
    clusters = some_clusters(rng, len(fr[0]), max_views)
    cam = gcam(K, 6 * voxel, 1)
    ctx.gain_enqueue(cam, poses, clusters)
    info, whole = ctx.gain_wait()
    assert info["n_views"] == max_views
    pick = rng.choice(max_views, 48, replace=False)
    _, want = G.gains(st, o, voxel, cam, poses[pick], clusters[pick], fr)
    assert whole[pick].tobytes() == want.tobytes()
    parts = []
    for a in range(0, max_views, 5000):
        ctx.gain_enqueue(cam, poses[a:a + 5000], clusters[a:a + 5000])
        parts.append(ctx.gain_wait()[1])
    assert np.concatenate(parts).tobytes() == whole.tobytes()
    with pytest.raises(capi.DsmError) as e:
        ctx.gain_enqueue(cam, np.concatenate([poses, poses[:1]]))
    assert e.value.code == -1
    ctx.close()


def test_stream_order():
    """A job reads the field and the frontier result it was enqueued behind, not the next field request or frontier
    job; clusters need a frontier job on the latest field request."""
    shape, voxel = (40, 30, 20), 0.2
    ctx = loader(shape, voxel)
    rng = np.random.default_rng(9)
    a = rng.choice(3, size=shape[::-1], p=(0.1, 0.1, 0.8)).astype(np.uint8)
    b = rng.choice(3, size=shape[::-1], p=(0.3, 0.1, 0.6)).astype(np.uint8)
    centre = G.centres([(20, 15, 10)], (0, 0, 0), voxel)[0]
    poses = [random_pose(rng, centre, 2.0) for _ in range(16)]
    cl = some_clusters(rng, 8, 16)
    cam = gcam(K, 10 * voxel, 1)
    ctx.debug_field_load_state(a, (0, 0, 0))
    with pytest.raises(capi.DsmError) as e:
        ctx.gain_enqueue(cam, poses, cl)                     # no frontier job on this field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    ctx.gain_enqueue(cam, poses, cl)                         # before the field is waited for
    with pytest.raises(capi.DsmError) as e:
        ctx.gain_enqueue(cam, poses)                         # one job in flight
    assert e.value.code == -7
    ctx.field_wait()
    fa = ctx.frontier_wait()
    got = ctx.gain_wait()
    want = G.gains(a, (0, 0, 0), voxel, cam, poses, cl, fa[:2])
    same(got, want, "first")
    ctx.frontier_enqueue(1)
    ctx.gain_enqueue(cam, poses, cl)
    ctx.debug_field_load_state(b, (5, 5, 5))                 # the next request, while the job is in flight
    got = ctx.gain_wait()
    ctx.field_wait()
    ctx.frontier_wait()
    same(got, want, "the old field")
    with pytest.raises(capi.DsmError) as e:
        ctx.gain_enqueue(cam, poses, cl)                     # the frontier job read the old field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    ctx.gain_enqueue(cam, poses, cl)
    fb = ctx.frontier_wait()
    ctx.frontier_enqueue(3)                                  # the next frontier job, while the gain job is in flight
    got = ctx.gain_wait()
    ctx.frontier_wait()
    same(got, G.gains(b, (5, 5, 5), voxel, cam, poses, cl, fb[:2]), "the old frontiers")
    ctx.field_enqueue((0, 0, 0), 1)                          # a plain request
    with pytest.raises(capi.DsmError) as e:
        ctx.gain_enqueue(cam, poses)
    assert e.value.code == -7
    ctx.field_wait()
    ctx.close()


def yaws_around(points):
    return [yaw_pose(k, p) for p in points for k in range(4)] + \
        [np.concatenate([yaw_pose(k, p).reshape(3, 4)[:, :3] @ _tilt(), np.asarray(p)[:, None]], axis=1).reshape(12)
         for p in points for k in range(4)]


def _tilt():
    a = np.deg2rad(45.0)
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])   # a yaw of 45 degrees in the camera


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_fields_of_the_drive(chunk, shape):
    """The windowed drive with loop-closure warps between calls; after every call a known field, its frontiers, a reach
    job from the camera to the clusters, and a gain job over eight yaws at each reached viewpoint and random poses,
    against the model on the field's own state grid; the same job on a resident twin of the request equals it."""
    lists = simple_lists()
    voxels = (0.125, 0.1, 0.3)
    ctxs, views = {}, {}
    for v in voxels:
        ctxs[v] = new_ctx(store=STORE)
        ctxs[v].field_enable(v, *shape)
        views[v] = Views(ctxs[v], 6)
        ctxs[v].frontier_enable(64, 1 << 16)
        ctxs[v].reach_enable(16, 1 << 12, 2048)
        ctxs[v].gain_enable(256)
    rng = np.random.default_rng(chunk)
    stored, seen = set(), 0
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for v in voxels:
            windowed(ctxs[v], t0, t1, lists, want_counts=False)
            views[v].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            for v in voxels:
                ctxs[v].pool_transform(warp(1))
                ctxs[v].inactive_transform(max(stored), warp(2))
                views[v].warp(warp(1))
        v = voxels[call % 3]
        ctx = ctxs[v]
        slots, poses = views[v].request()
        cam = camera(t1 - 1)
        ctx.field_enqueue_known(cam, 5, slots, poses)
        _, origin, _ = ctx.field_wait()
        state, _ = ctx.field_state()
        ctx.frontier_enqueue(1 + call % 3)
        fc, fv, _ = ctx.frontier_wait()
        ctx.reach_enqueue(cam, 0.0, 1, None, True)
        _, targets, _, _ = ctx.reach_wait()
        vp = targets["viewpoint"][targets["status"] == 0][:3]
        nz, ny, nx = state.shape
        pts = G.centres(np.stack([vp % nx, vp // nx % ny, vp // (nx * ny)], 1), origin, v) if len(vp) else np.zeros((0, 3))
        gp = yaws_around(list(pts) + [cam]) + [random_pose(rng, cam, 2.0) for _ in range(8)]
        ub = call % 2
        gc = gcam(K, (10 + 7 * (call % 3)) * np.float32(v), ub)
        with_clusters = call % 3 != 1
        cl = (np.arange(len(gp)) % (len(fc) + 2) - 1).astype(np.int32) if with_clusters else None
        ctx.gain_enqueue(gc, gp, cl)
        got = ctx.gain_wait()
        same(got, G.gains(state, origin, v, gc, gp, cl, (fc, fv)), f"frames {t0}-{t1 - 1}, voxel {v}")
        seen += int((got[1]["n_free"] > 0).sum()) > 1
        # a resident twin of the same request
        ctx.field_enqueue_known(cam, 5, slots, poses, host_copy=False)
        ctx.field_wait()
        if with_clusters:
            ctx.frontier_enqueue(1 + call % 3)
            ctx.frontier_wait()
        ctx.gain_enqueue(gc, gp, cl)
        twin = ctx.gain_wait()
        assert twin[0].tobytes() == got[0].tobytes() and twin[1].tobytes() == got[1].tobytes(), "resident twin"
    assert seen > 0 or shape == (1, 1, 1)
    for c in ctxs.values():
        c.close()


def test_gain_jobs_change_nothing_else(tmp_path):
    """A drive with frontier, reach and gain jobs beside a publish snapshot and an asynchronous checkpoint leaves the
    map, both published clouds, the fields, the state grids, the frontiers, the reach results and the checkpoint files
    byte-identical to a twin without gain jobs."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    va, vb = {}, {}
    for c, d in ((a, va), (b, vb)):
        c.field_enable(voxel, *shape)
        c.publish_enable()
        c.checkpoint_enable()
        d["v"] = Views(c, 4)
        c.frontier_enable(32, 4096)
        c.reach_enable(16, 1 << 12, 1024)
    a.gain_enable(64)
    rng = np.random.default_rng(5)
    stored = set()
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        for c, d in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            d["v"].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        outs = []
        gp = [random_pose(rng, camera(t1 - 1), 1.0) for _ in range(24)]
        gc = gcam(K, 20 * voxel, call % 2)
        for c, d in ((a, va), (b, vb)):
            slots, poses = d["v"].request()
            c.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
            c.frontier_enqueue(1)
            c.reach_enqueue(camera(t1 - 1), 0.1, 2, [camera(0)], True)
            if c is a:
                a.gain_enqueue(gc, gp, np.arange(24, dtype=np.int32) - 1)
            c.publish_enqueue(5)
            c.checkpoint_enqueue(str(tmp_path / f"{'ab'[c is b]}{call}.dsm"))
            if call % 2 == 1 and stored:
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
                d["v"].warp(warp(1))
            f = c.field_wait()
            st = c.field_state()
            fr = c.frontier_wait()
            re = c.reach_wait()
            p = c.publish_wait()
            assert c.checkpoint_wait(True)
            outs.append((f, st, p, fr, re))
        got = a.gain_wait()
        what = f"after frames {t0}-{t1 - 1}"
        same(got, G.gains(outs[0][1][0], outs[0][0][1], voxel, gc, gp, np.arange(24) - 1, outs[0][3][:2]), what)
        fa, fb = outs[0][0], outs[1][0]
        assert fa[0].tobytes() == fb[0].tobytes() and outs[0][1][0].tobytes() == outs[1][1][0].tobytes(), f"{what}: field"
        assert all(x.tobytes() == y.tobytes() for x, y in zip(outs[0][3], outs[1][3])), f"{what}: frontiers"
        assert all(x.tobytes() == y.tobytes() for x, y in zip(outs[0][4][:3], outs[1][4][:3])), f"{what}: reach"
        assert outs[0][2][0].tobytes() == outs[1][2][0].tobytes() and outs[0][2][1].tobytes() == outs[1][2][1].tobytes(), f"{what}: clouds"
        assert map_state(a) == map_state(b), f"{what}: map"
        assert filecmp.cmp(str(tmp_path / f"a{call}.dsm"), str(tmp_path / f"b{call}.dsm"), shallow=False), f"{what}: checkpoint"
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_wait():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    views = Views(b, 4)
    b.gain_enable(8)
    for call, t0 in enumerate(range(0, first + 2)):
        windowed(b, t0, t0 + 1, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 1)
    slots, poses = views.request()
    b.field_enqueue_known(camera(first - 1), 1, slots, poses)
    gp = [yaw_pose(k, camera(first - 1)) for k in range(4)]
    gc = gcam(K, 30 * voxel, 0)
    b.gain_enqueue(gc, gp)
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6
    _, origin, _ = e.value.field
    state, _ = b.field_state()
    with pytest.raises(capi.DsmError) as e:
        b.gain_wait()
    assert e.value.code == -6
    same(e.value.gain, G.gains(state, origin, voxel, gc, gp), "rejected")
    assert e.value.gain[1]["n_free"].sum() > 0
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    b.close()


def test_error_contract():
    lib = capi.load_library()
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    st = np.full((4, 5, 6), FREE, np.uint8)
    ok = capi.DsmGainCamera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    pose = np.eye(3, 4).reshape(1, 12)
    P = pose.ctypes.data
    assert lib.dsm_gain_enable(ctx.h, 1) == -7                            # before dsm_field_enable
    ctx.field_enable(0.2, 6, 5, 4)
    assert lib.dsm_gain_enable(ctx.h, 1) == -7                            # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, None, 1) == -7   # before dsm_gain_enable
    assert lib.dsm_gain_wait(ctx.h, None, None) == -7
    for n in (0, -1, G.MAX_VIEWS + 1):
        assert lib.dsm_gain_enable(ctx.h, n) == -1, n
    assert lib.dsm_gain_enable(None, 1) == -1
    ctx.gain_enable(128)
    assert lib.dsm_gain_enable(ctx.h, 1) == -7                            # once
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, None, 1) == -7   # no field request yet
    assert lib.dsm_gain_wait(ctx.h, None, None) == -7                     # nothing enqueued
    ctx.field_enqueue((0, 0, 0), 1)                                       # a plain request
    ctx.field_wait()
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, None, 1) == -7
    load_known(ctx, st, (0, 0, 0), 0.2)
    cl = np.zeros(1, np.int32)
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, cl.ctypes.data, 1) == -7   # clusters without a frontier job
    nan, inf = float("nan"), float("inf")
    bad = []
    for field, value in [("fx", 0.0), ("fx", -1.0), ("fx", nan), ("fy", inf), ("cx", nan), ("cy", inf), ("width", 0), ("width", 65537),
                         ("height", 0), ("height", 65537), ("max_range", 0.0), ("max_range", -1.0), ("max_range", nan),
                         ("max_range", inf), ("max_range", 25.7), ("unknown_blocks", 2), ("unknown_blocks", -1)]:
        c = capi.DsmGainCamera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
        setattr(c, field, value)
        bad.append((ctypes.byref(c), P, None, 1))
    p2 = pose.copy()
    p2[0, 7] = nan
    bad += [(ctypes.byref(ok), p2.ctypes.data, None, 1), (ctypes.byref(ok), P, None, -1),
            (ctypes.byref(ok), np.tile(pose, (129, 1)).ctypes.data, None, 129),
            (ctypes.byref(ok), None, None, 1), (None, P, None, 1)]
    for args in bad:
        assert lib.dsm_gain_enqueue(ctx.h, *args) == -1, args
    assert lib.dsm_gain_enqueue(None, ctypes.byref(ok), P, None, 1) == -1
    ctx.frontier_enable(4, 64)
    ctx.frontier_enqueue(1)
    ctx.frontier_wait()
    cl2 = np.array([-2], np.int32)
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, cl2.ctypes.data, 1) == -1
    # the work bound at 128 v: 123 views of (2 * 128 + 3)^3 voxels pass, 124 do not
    far = capi.DsmGainCamera(10.0, 10.0, 5.0, 5.0, 10, 10, 25.6, 1)
    assert (123 * 259 ** 3 <= G.MAX_WORK) and (124 * 259 ** 3 > G.MAX_WORK)
    P124 = np.tile(pose, (124, 1))
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(far), P124.ctypes.data, None, 124) == -1
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(far), P124.ctypes.data, None, 123) == 0
    info, g = ctx.gain_wait()
    assert info["n_views"] == 123 and (g["status"] == 0).all()
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, cl.ctypes.data, 1) == 0
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), P, None, 1) == -7   # one job in flight
    info = np.zeros(1, capi.GAIN_INFO_DTYPE)
    assert lib.dsm_gain_wait(ctx.h, info.ctypes.data, None) == 0
    assert info[0]["n_views"] == 1 and info[0]["n_clusters_table"] == 0 and info[0]["reserved"].tolist() == [0, 0]
    assert lib.dsm_gain_wait(ctx.h, None, None) == -7
    assert lib.dsm_gain_enqueue(ctx.h, ctypes.byref(ok), None, None, 0) == 0   # no views
    info, g = ctx.gain_wait()
    assert info["n_views"] == 0 and len(g) == 0
    ctx.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)
MAX_VIEWS = 5
RELOAD = 12   # the node saves and loads its state after this depth message


def test_node_view_gain_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers() and view_gain() at eight yaws
    with named clusters equal the model over the grid, frontiers and poses the driver dumps; clouds, PLY and PCD files
    equal a twin without gain jobs; view_gain() with clusters before a frontiers() call on the frame, and after
    load_state until the next fused frame, returns DSM_E_STATE."""
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    node = [2, 0, 1 << 20, 1 << 21, *FIELD, MAX_VIEWS, MAX_RANGE]
    r = run_driver("gain_main", str(tmp_path), cam, sc, node + [64, RELOAD], tag="a", after=[pa])
    q = run_driver("gain_main", str(tmp_path), cam, sc, node + [0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, ub = r.i(), r.i()
        max_range = float(r.take(np.float32, 1)[0])
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        poses, named = r.lst(np.float64).reshape(-1, 12), r.lst(np.int32)
        info = r.take(np.uint8, G.INFO_DTYPE.itemsize).view(G.INFO_DTYPE)[0].copy()
        gains = r.lst(G.GAIN_DTYPE)
        before, after_load = r.i(), r.i()
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == 0 and rr == 0 and rq == 0, f"message {t}: {rc} {rr} {rq}"
        gc = G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, max_range, ub)
        same((info, gains), G.gains(state, origin, voxel, gc, poses, named, (clusters, vox)), f"message {t}")
        found += int((gains["n_free"] > 0).sum()) > 0
        assert before == -7, f"message {t}: view_gain() before frontiers()"
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: view_gain() after load_state"
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
    assert found > 0
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
