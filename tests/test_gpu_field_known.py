"""dsm_views_enable / _capture, dsm_field_enqueue_known and dsm_field_state: free versus unknown space, and the distance
to anything not known to be free.

Every known field equals oracle/pyoracle_field_known applied to the synchronous readers (dsm_pool_export_cloud(m) +
dsm_inactive_export_cloud) and to the rays of dsm_get_seeds of every captured frame, at the poses the test passes, bit
for bit in the state grid, the distance grid, n_occupied and n_free; the geometry of the synthetic scene; captures
change nothing in the map, the plain fields or the published clouds; a known field beside a publish snapshot and an
asynchronous checkpoint, and a query on it; the rejected-frame and error contracts; and a size a user runs.  The node is
checked through tests/cpp/field_known_main.cpp."""
import filecmp

import numpy as np
import pytest

import pyoracle_field
import pyoracle_field_known
import pyoracle_field_query
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SEED_DTYPE, SURFEL_DTYPE
from known_space import (K, MAX_RANGE, MAX_VIEWS, NODE_FIELD, RELOAD, SMALL_CAM, Views, assert_error_stays, node_args, pose12,
                         rejected_known, twin_clouds, twin_node_tail)
from node_drive import node_script, run_driver
from resident_map import SHAPES, STORE, T, camera, field_points, frames, map_state, new_ctx, simple_lists, warp, windowed, xyz

pytestmark = pytest.mark.gpu

def known_equals_oracle(ctx, views, voxel, shape, center, m, what, host_copy=True, slots=None):
    all_slots, poses = views.request()
    if slots is not None:
        keep = [all_slots.index(s) for s in slots]
        all_slots, poses = slots, poses[keep]
    ctx.field_enqueue_known(center, m, all_slots, poses, host_copy=host_copy)
    dist, origin, n_occ = ctx.field_wait()
    state, n_free = ctx.field_state()
    want = pyoracle_field_known.known_field(field_points(ctx, m), voxel, shape, center, views.oracle_views(all_slots), MAX_RANGE)
    assert origin.tolist() == want[1].tolist(), f"{what}: origin"
    assert (n_occ, n_free) == (want[2], want[4]), f"{what}: occupied / free {n_occ} / {n_free}, want {want[2]} / {want[4]}"
    if host_copy:
        assert state.tobytes() == want[3].tobytes(), f"{what}: {(state != want[3]).sum()} states differ"
        assert dist.tobytes() == want[0].tobytes(), f"{what}: {(dist.view(np.uint32) != want[0].view(np.uint32)).sum()} distances differ"
    else:
        assert dist is None and state is None
    return want


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_field_equals_the_oracle(chunk, shape):
    """The windowed drive with loop-closure warps between calls, the views warped with the map; after every call one
    known field, the voxel edge cycling through 0.125, 0.1 and 0.3 and host copy and resident alternating.  Six slots:
    later frames overwrite the earliest."""
    lists = simple_lists()
    voxels = (0.125, 0.1, 0.3)
    ctxs, views = {}, {}
    for v in voxels:
        ctxs[v] = new_ctx(store=STORE)
        ctxs[v].field_enable(v, *shape)
        views[v] = Views(ctxs[v], 6)
    stored, seen = set(), {"free": 0, "occupied": 0, "unknown": 0}
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
        want = known_equals_oracle(ctxs[v], views[v], v, shape, camera(t1 - 1), 5, f"frames {t0}-{t1 - 1}, voxel {v}",
                                   host_copy=call % 2 == 0)
        seen["free"] += want[4] > 0
        seen["occupied"] += want[2] > 0
        seen["unknown"] += int((want[3] == 0).sum()) > 0
    # a one-voxel grid centred on the camera is carved by the camera's own rays: never unknown, and no surface in it
    assert all(seen.values()) if shape != (1, 1, 1) else seen["free"], seen
    # a subset of the slots, in another order, and none
    v = voxels[0]
    slots = sorted(views[v].rays)
    known_equals_oracle(ctxs[v], views[v], v, shape, camera(T - 1), 1, "reversed subset", slots=slots[::-2])
    want = known_equals_oracle(ctxs[v], views[v], v, shape, camera(T - 1), 1, "no views", slots=[])
    assert want[4] == 0 and (want[0] == 0).all()
    for c in ctxs.values():
        c.close()


def test_geometry_of_the_synthetic_scene():
    """The voxels on the line from the last camera to the centre of the next box's front face are free up to the box;
    the voxels 1 m below the ground plane (y = 1.65 m, y down) are unknown; known <= plain everywhere.  (The road
    straight ahead ends at a backdrop beyond the camera's far limit, whose seeds give no rays: it stays unknown.)"""
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    voxel, shape = 0.2, (64, 32, 64)
    ctx.field_enable(voxel, *shape)
    views = Views(ctx, T)
    for call, t0 in enumerate(range(0, T, 4)):
        windowed(ctx, t0, t0 + 4, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 4)
    c = camera(T - 1)
    want = known_equals_oracle(ctx, views, voxel, shape, c, 5, "end of the drive")
    state, o = want[3], want[1].astype(np.int64)
    face = np.array([2.5, 1.15, 8.0 * np.ceil((c[2] - 5.0) / 8.0) + 5.0])   # the centre of the next box's front face
    L = np.linalg.norm(face - c)
    to_box = [c + s * (face - c) / L for s in np.arange(0.2, L - 0.3, 0.05)]

    def at(p):
        q = np.floor(np.asarray(p) / np.float64(np.float32(voxel))).astype(np.int64) - o
        return state[q[2], q[1], q[0]]
    assert len(to_box) > 10
    assert [int(at(p)) for p in to_box] == [pyoracle_field_known.FREE] * len(to_box)
    below = [np.array([c[0] + dx, 2.65, c[2] + dz]) for dx in (-2.0, 0.0, 2.0) for dz in (1.0, 3.0, 5.0)]
    assert [int(at(p)) for p in below] == [pyoracle_field_known.UNKNOWN] * len(below)
    plain = pyoracle_field.field(field_points(ctx, 5), voxel, shape, c)
    assert (want[0] <= plain[0]).all() and want[2] == plain[2]
    ctx.close()


@pytest.mark.parametrize("chunk", [1, 4])
def test_views_change_nothing_else(chunk):
    """A context that captures every frame and requests known fields gives byte-identical plain fields, map and
    published clouds to a twin without views."""
    lists = simple_lists()
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    shape, voxel = (64, 64, 32), 0.1
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.publish_enable()
    va = Views(a, 4)
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c in (a, b):
            windowed(c, t0, t1, lists, want_counts=False)
        va.capture_call(call, t0, t1)
        slots, poses = va.request()
        a.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
        a.field_wait()
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            for c in (a, b):
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
        for c in (a, b):
            c.field_enqueue(camera(t1 - 1), 5)
        fa, fb = a.field_wait(), b.field_wait()
        for c in (a, b):
            c.publish_enqueue(5)
        pa, pb = a.publish_wait(), b.publish_wait()
        what = f"after frames {t0}-{t1 - 1}"
        assert fa[0].tobytes() == fb[0].tobytes() and fa[2] == fb[2], f"{what}: plain field"
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes(), f"{what}: published clouds"
        assert map_state(a) == map_state(b), f"{what}: pool, store or table"
        with pytest.raises(capi.DsmError) as e:   # the last waited request was a plain one
            a.field_state()
        assert e.value.code == -7
    a.close()
    b.close()


def test_known_field_beside_a_snapshot_a_checkpoint_and_a_query(tmp_path):
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    shape, voxel = (64, 64, 32), 0.125
    ctx.field_enable(voxel, *shape)
    ctx.field_query_enable(4096, 0, 0)
    ctx.publish_enable()
    ctx.checkpoint_enable()
    views = Views(ctx, 8)
    for call, t0 in enumerate(range(0, 10, 2)):
        windowed(ctx, t0, t0 + 2, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 2)
    slots, poses = views.request()
    ctx.publish_enqueue(5)
    ctx.checkpoint_enqueue(str(tmp_path / "async.dsm"))
    ctx.field_enqueue_known(camera(9), 5, slots, poses, host_copy=False)
    rng = np.random.default_rng(5)
    o = pyoracle_field.origin(camera(9), voxel, shape)
    pts = (o + rng.uniform(-0.5, np.array(shape) + 0.5, (4096, 3))) * np.float64(np.float32(voxel))
    ctx.field_query_enqueue(pts)
    ctx.inactive_transform(1, warp(2))   # enqueued behind all of them: none sees it
    ctx.pool_transform(warp(1))
    dist, origin, n_occ = ctx.field_wait()
    state, n_free = ctx.field_state()
    samples, _ = ctx.field_query_wait()
    active, inactive, _ = ctx.publish_wait()
    assert ctx.checkpoint_wait(True)
    ref = new_ctx(store=STORE)
    for t0 in range(0, 10, 2):
        windowed(ref, t0, t0 + 2, lists, want_counts=False)
    want = pyoracle_field_known.known_field(field_points(ref, 5), voxel, shape, camera(9), views.oracle_views(slots), MAX_RANGE)
    assert dist is None and state is None and (n_occ, n_free) == (want[2], want[4]) and origin.tolist() == want[1].tolist()
    q = pyoracle_field_query.sample(want[0], want[1], voxel, pts)
    assert samples.tobytes() == q.tobytes()
    assert want[4] > 0 and int((want[3] == 0).sum()) > 0
    assert active.tobytes() == ref.pool_export_cloud(5).tobytes() and inactive.tobytes() == ref.inactive_export_cloud().tobytes()
    ref.map_save(str(tmp_path / "sync.dsm"))
    assert filecmp.cmp(str(tmp_path / "async.dsm"), str(tmp_path / "sync.dsm"), shallow=False)
    ctx.close()
    ref.close()


def test_rejected_frame_comes_back_from_wait():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    a = new_ctx(store=STORE)
    for t0 in range(0, first, 1):
        windowed(a, t0, t0 + 1, lists, want_counts=False)
    r = rejected_known(lambda ctx: None, lambda ctx, first: None)
    want = pyoracle_field_known.known_field(field_points(a, 1), r.voxel, r.shape, camera(first - 1), r.views.oracle_views(r.slots),
                                            MAX_RANGE)
    assert r.field[0].tobytes() == want[0].tobytes() and r.field[2] == want[2] and want[2] > 0
    assert r.state.tobytes() == want[3].tobytes() and r.n_free == want[4] > 0
    assert_error_stays(r.ctx)
    a.close()
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    C = (capi.ctypes.c_double * 3)
    I = capi.ctypes.c_int32

    def known(ctx, slots, poses, n=None, center=(0, 0, 0), m=5):
        s = np.ascontiguousarray(slots, np.int32)
        p = np.ascontiguousarray(poses, np.float64)
        return lib.dsm_field_enqueue_known(ctx.h, C(*center), m, s.ctypes.data if s.size else None,
                                           p.ctypes.data if p.size else None, len(s) if n is None else n, 1)

    ctx = new_ctx(store=STORE)
    assert lib.dsm_views_enable(ctx.h, 4, 10.0) == -7                      # before dsm_field_enable
    ctx.field_enable(0.1, 16, 16, 8)
    assert lib.dsm_views_capture(ctx.h, 0, 0) == -7                        # before dsm_views_enable
    assert known(ctx, [], []) == -7
    assert lib.dsm_field_state(ctx.h, None, None) == -7
    for mv, r in [(0, 10.0), (65537, 10.0), (-1, 10.0), (4, 0.0), (4, -1.0), (4, float("nan")), (4, float("inf")), (4, 102.5)]:
        assert lib.dsm_views_enable(ctx.h, mv, r) == -1, (mv, r)
    assert lib.dsm_views_enable(None, 4, 10.0) == -1
    assert lib.dsm_views_enable(ctx.h, 4, 102.4) == 0                      # 1024 voxels exactly
    assert lib.dsm_views_enable(ctx.h, 4, 10.0) == -7                      # once
    assert lib.dsm_views_capture(ctx.h, 0, 0) == -7                        # no call has taken images
    windowed(ctx, 0, 2, simple_lists(), want_counts=False)
    for f, s in [(0, -1), (0, 4), (-1, 0), (2, 0)]:
        assert lib.dsm_views_capture(ctx.h, f, s) == -1, (f, s)
    assert lib.dsm_views_capture(None, 0, 0) == -1
    assert lib.dsm_views_capture(ctx.h, 1, 2) == 0
    P = pose12(frames()[1][0])
    assert known(ctx, [0], [P]) == -1                                      # never captured
    assert known(ctx, [-1], [P]) == -1 and known(ctx, [4], [P]) == -1
    assert known(ctx, [2] * 5, [P] * 5) == -1                             # more than max_views
    assert known(ctx, [2], [P], n=-1) == -1
    assert lib.dsm_field_enqueue_known(ctx.h, C(0, 0, 0), 5, None, None, 1, 1) == -1
    for k in range(12):
        bad = P.copy()
        bad[k] = [np.nan, np.inf, -np.inf][k % 3]
        assert known(ctx, [2], [bad]) == -1, k
    assert known(ctx, [2], [P], m=0) == -1
    assert known(ctx, [2], [P], center=(np.nan, 0, 0)) == -1
    with pytest.raises(ValueError):                                        # the binding checks the pose count
        ctx.field_enqueue_known((0, 0, 0), 5, [2, 2], [P])
    assert known(ctx, [2, 2], [P, P]) == 0                                 # one slot twice is two views
    assert known(ctx, [2], [P]) == -7                                      # one field in flight
    assert lib.dsm_field_enqueue(ctx.h, C(0, 0, 0), 5) == -7
    assert lib.dsm_field_state(ctx.h, None, None) == -7                    # not waited yet
    dist, origin, n_occ = ctx.field_wait()
    n_free = I(-1)
    assert lib.dsm_field_state(ctx.h, None, capi.ctypes.byref(n_free)) == 0 and n_free.value >= 0
    assert lib.dsm_field_state(None, None, None) == -1
    ctx.debug_stop_after(2)                                                # the schedule stops before the plane fit
    windowed(ctx, 2, 3, simple_lists(), want_counts=False)
    assert lib.dsm_views_capture(ctx.h, 0, 1) == -7
    ctx.close()


def test_the_most_views_one_request_takes():
    """DSM_VIEWS_MAX views of 64x48 frames in one request: one fused frame captured into every slot, the views at seven
    poses, the last view alone at the seventh, and one view whose rotation overflows R * p (an infinite ray length
    cuts its rays to zero length; a ray with an infinite or NaN endpoint coordinate carves nothing).  Equal to the
    oracle over the distinct views, and the last view carves voxels no other does."""
    cam = SMALL_CAM
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=1 << 14)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    voxel, shape, max_range = 0.1, (64, 64, 64), 5.0
    ctx.field_enable(voxel, *shape)
    n = pyoracle_field_known.VIEWS_MAX
    ctx.views_enable(n, max_range)
    gray, depth = synth.make_frame(cam, 77, synth.pose_stream(0))
    ctx.fuse_stream_resident([0], gray[None], depth[None], synth.pose_stream(0)[None])
    rays = pyoracle_field_known.capture(ctx.seeds(0))   # the first run uses frame slot 0
    for j in range(n):
        ctx.views_capture(0, j)
    base = pose12(synth.pose_stream(0))
    kinds = []
    for k in range(6):
        P = base.copy()
        P[3] += 0.3 * k
        kinds.append(P)
    last = base.copy()
    last[7] -= 1.5                                      # 1.5 m higher (y down)
    huge = base.copy()
    huge[0] = 1.7e308                                   # R_00: R * p overflows for |p_x| > 1.06
    kind = [j % 6 for j in range(n)]
    kind[100], kind[n - 1] = 7, 6
    table = kinds + [last, huge]
    poses = np.array([table[k] for k in kind])
    c = base[[3, 7, 11]]
    ctx.field_enqueue_known(c, 1, list(range(n)), poses)
    dist, origin, n_occ = ctx.field_wait()
    state, n_free = ctx.field_state()
    want = pyoracle_field_known.known_field(xyz(ctx.pool_export_cloud(1)), voxel, shape, c, [(rays, P) for P in table], max_range)
    assert origin.tolist() == want[1].tolist() and (n_occ, n_free) == (want[2], want[4])
    assert state.tobytes() == want[3].tobytes() and dist.tobytes() == want[0].tobytes()
    without_last = pyoracle_field_known.known_field(xyz(ctx.pool_export_cloud(1)), voxel, shape, c, [(rays, P) for P in kinds + [huge]], max_range)
    assert without_last[4] < n_free
    a, b, _ = pyoracle_field_known.segments(rays, huge, max_range)
    assert not np.isfinite(b).all() and np.isfinite(b).all(axis=1).any()   # both kinds of overflowing ray occur
    ctx.close()


def test_a_size_a_user_runs():
    """320x320x40 at 0.2 m over 256 views of 1226x370 frames: eight frames fused once, each captured into 32 slots,
    at 256 poses spread along and across the road."""
    cam = K
    ctx = capi.Context(cam, max_batch=16, max_local_surfels=1 << 18)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    shape, voxel = (320, 320, 40), 0.2
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(256, MAX_RANGE)
    imgs = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(8)]
    ctx.fuse_stream_resident(list(range(8)), np.stack([g for g, _ in imgs]), np.stack([d for _, d in imgs]),
                             np.stack([synth.pose_stream(t) for t in range(8)]))
    rays = [pyoracle_field_known.capture(ctx.seeds(f)) for f in range(8)]   # one run of 8 frames: slots 0..7
    slots, poses, views = [], [], []
    for j in range(256):
        f = j % 8
        ctx.views_capture(f, j)
        P = pose12(synth.pose_stream(f))
        P[3] += 0.35 * (j // 8 % 8) - 1.2
        P[11] += 0.8 * (j // 64)
        slots.append(j)
        poses.append(P)
        views.append((rays[f], P))
    c = pose12(synth.pose_stream(4))[[3, 7, 11]]
    ctx.field_enqueue_known(c, 1, slots, np.array(poses))
    dist, origin, n_occ = ctx.field_wait()
    state, n_free = ctx.field_state()
    want = pyoracle_field_known.known_field(xyz(ctx.pool_export_cloud(1)), voxel, shape, c, views, MAX_RANGE)
    assert origin.tolist() == want[1].tolist() and (n_occ, n_free) == (want[2], want[4])
    assert state.tobytes() == want[3].tobytes() and dist.tobytes() == want[0].tobytes()
    assert n_free > 10000 and n_occ > 0
    ctx.close()


# ---- the node ----
def test_node_known_space_equals_the_oracle_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): every fused frame's known field equals the oracle over the views the
    node carried (the driver dumps their frames' seeds and current poses); clouds, PLY and PCD files equal a twin
    without known space; after load_state the slot table is empty and refills."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("field_known_main", str(tmp_path), cam, sc, node_args() + [RELOAD], tag="a", after=[pa])
    q = run_driver("field_known_main", str(tmp_path), cam, sc, node_args(0) + [RELOAD], tag="b", after=[pb])
    free, most = 0, 0
    for t in range(n):
        rc = r.i()
        c = r.take(np.float64, 3).copy()
        origin, n_occ = r.take(np.int32, 3).copy(), r.i()
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        state, n_free = r.lst(np.uint8).reshape(nz, ny, nx), r.i()
        views = []
        for _ in range(r.i()):
            seeds = r.lst(SEED_DTYPE)
            views.append((pyoracle_field_known.capture(seeds), r.lst(np.float64).copy()))
        act, inact = twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}"
        assert 1 <= len(views) <= MAX_VIEWS
        if t == RELOAD:
            assert len(views) == 1, "the slot table refills from empty after load_state"
        most = max(most, len(views))
        want = pyoracle_field_known.known_field(xyz(act, inact), voxel, (nx, ny, nz), c, views, MAX_RANGE)
        assert origin.tolist() == want[1].tolist() and (n_occ, n_free) == (want[2], want[4]), f"message {t}"
        assert state.tobytes() == want[3].tobytes() and dist.tobytes() == want[0].tobytes(), f"message {t}"
        free += n_free > 0
    assert free > n // 2 and most > 2
    twin_node_tail(r, q, pa, pb)
