"""dsm_trajectory_enable / _enqueue / _wait: B-spline trajectories optimised on the device against the signed grid.

The optimised control points, the records and the header equal oracle/pyoracle_trajectory bit for bit on crafted state
grids loaded through dsm_debug_field_load_state (a pillar, a wall with a gap, a block of unknown space, random states,
and both infinity rules), with 7 to 256 points per trajectory, 1 to max_trajectories trajectories, memory 1 and 16 and
points that leave the grid, and on the windowed drive's plain and known fields.  The final check agrees with signed
point queries of the model's samples; a job in flight across the next field request reads the old grid; a drive with
trajectory jobs leaves the map, the fields and the published clouds byte-identical to a twin's without them.  The
rejected-frame and error contracts, and dsm::SurfelMapNode (tests/cpp/trajectory_main.cpp)."""
import numpy as np
import pytest

import pyoracle_field_known
import pyoracle_field_signed as fs
import pyoracle_trajectory as tj
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from densesurfelmapping_b200.elements import POINT_DTYPE
from node_drive import node_script, run_driver
from resident_map import STORE, T, camera, field_points, map_state, new_ctx, simple_lists, warp, windowed, xyz
from test_gpu_field_known import MAX_RANGE, Views

pytestmark = pytest.mark.gpu

SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
UNKNOWN, OCCUPIED, FREE = 0, 1, 2
CAPS = (64, 1 << 14, 16)


def known_ctx(shape, voxel):
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(1, 1.0)
    ctx.field_signed_enable()
    ctx.trajectory_enable(*CAPS)
    ctx.field_query_enable(1 << 16, 1, 2)
    return ctx


def random_trajectories(rng, origin, voxel, shape, n, lens=None):
    """n trajectories of 7 to 256 points: seeded random walks through and beyond the grid's box."""
    v = float(np.float32(voxel))
    lo, size = np.asarray(origin, np.float64) * v, np.array(shape, np.float64) * v
    lens = rng.integers(7, 257, n) if lens is None else np.asarray(lens)
    pts = []
    for N in lens:
        a, b = lo + rng.random(3) * size, lo + rng.random(3) * size
        t = np.linspace(0, 1, N)[:, None]
        q = a + t * (b - a) + rng.standard_normal((N, 3)) * v * rng.uniform(0.1, 3)
        pts.append(q)
    ofs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    dt = rng.uniform(0.05, 1.0, n)
    return np.concatenate(pts), ofs, dt


def equals_the_model(ctx, pts, ofs, dt, p, sdist, origin, voxel, what):
    ctx.trajectory_enqueue(pts, ofs, dt, p)
    info, rec, out = ctx.trajectory_wait()
    wq, wr, wi = tj.job(pts, ofs, dt, p, sdist, origin, voxel)
    assert info.tobytes() == wi.tobytes(), f"{what}: header {info} != {wi}"
    bad = [k for k in range(len(rec)) if rec[k].tobytes() != wr[k].tobytes()]
    assert not bad, f"{what}: records {bad[:5]} differ, e.g. {rec[bad[0]]} != {wr[bad[0]]}"
    assert out.tobytes() == wq.tobytes(), f"{what}: {int((out != wq).any(1).sum())} points differ"
    return info, rec, out


def final_check_equals_signed_queries(ctx, out, ofs, rec, p):
    """min_dist, argmin and first_hit of every record against signed point queries of the model's samples."""
    for j in range(len(ofs) - 1):
        s = tj.curve_samples(out[ofs[j]:ofs[j + 1]], p["samples"])
        ctx.field_query_enqueue(s, signed=True)
        d = ctx.field_query_wait()[0]["dist"]
        inside = ~np.isnan(d)
        assert int((~inside).sum()) == rec[j]["n_outside"]
        if inside.any():
            m = d[inside].min()
            assert np.float32(m).tobytes() == rec[j]["min_dist"].tobytes()
            assert rec[j]["argmin"] == np.flatnonzero(inside & (d == m))[0]
        hits = np.flatnonzero(inside & (d < np.float32(p["radius"])))
        assert rec[j]["first_hit"] == (hits[0] if len(hits) else -1)


def crafted_grids(shape, rng):
    nx, ny, nz = shape
    grids = {"free": np.full(shape[::-1], FREE, np.uint8), "unknown": np.full(shape[::-1], UNKNOWN, np.uint8)}
    st = np.full(shape[::-1], FREE, np.uint8)
    st[:, ny // 2 - 2:ny // 2 + 2, nx // 2 - 2:nx // 2 + 2] = OCCUPIED
    grids["pillar"] = st
    st = np.full(shape[::-1], FREE, np.uint8)
    st[:, :, nx // 2 - 1:nx // 2 + 1] = OCCUPIED
    st[nz // 3:2 * nz // 3, ny // 3:2 * ny // 3, nx // 2 - 1:nx // 2 + 1] = FREE
    grids["wall"] = st
    st = np.full(shape[::-1], FREE, np.uint8)
    st[:, ny // 3:, nx // 3:2 * nx // 3] = UNKNOWN
    grids["unknown_block"] = st
    grids["random"] = rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1], p=[0.2, 0.1, 0.7]).astype(np.uint8)
    return grids


@pytest.mark.parametrize("memory", [1, 16])
def test_crafted_grids_equal_the_model(memory):
    shape, voxel, origin = (48, 32, 16), 0.1, (-24, -16, -8)
    rng = np.random.default_rng(memory)
    ctx = known_ctx(shape, voxel)
    p = tj.params(1, 20, 1, margin=0.3, v_max=3.0, a_max=6.0, max_iter=60, memory=memory, max_ls=12, samples=6, radius=0.15)
    for name, st in crafted_grids(shape, rng).items():
        ctx.debug_field_load_state(st, origin)
        ctx.field_wait()
        sdist = ctx.field_signed()
        assert sdist.tobytes() == fs.state_field(st, voxel)[1].tobytes()
        for n in (1, 5, CAPS[0]):
            pts, ofs, dt = random_trajectories(rng, origin, voxel, shape, n, [7, 256, 64, 9, 33][:n] if n < CAPS[0] else None)
            if ofs[-1] > CAPS[1]:
                continue
            info, rec, out = equals_the_model(ctx, pts, ofs, dt, p, sdist, origin, voxel, f"{name} n={n}")
            if name == "unknown":
                assert (rec["status"] == 3).all() and out.tobytes() == pts.tobytes()
            elif name == "free":
                assert (rec["clearance"] == 0).all()
            if n == 5:
                final_check_equals_signed_queries(ctx, out, ofs, rec, p)
        # the hand cases: straight paths through the obstacle, and max_iter = 0
        for p2 in (p, dict(p, max_iter=0)):
            line = np.linspace([-2.0, 0.15, 0.0], [2.0, 0.15, 0.0], 24)
            q = np.concatenate([line[:1]] * 2 + [line] + [line[-1:]] * 2)
            equals_the_model(ctx, q, [0, len(q)], [0.5], p2, sdist, origin, voxel, f"{name} line max_iter={p2['max_iter']}")
    ctx.close()


def reach_paths(ctx, start, origin, voxel, shape, rng):
    """The voxel-centre paths of a reach job from `start` to random goals in the latest known field, in world metres."""
    v = float(np.float32(voxel))
    goals = (rng.integers(0, shape, (24, 3)) + np.asarray(origin) + 0.5) * v
    ctx.reach_enqueue(start, 0.2, 1, goals)
    _, targets, path, _ = ctx.reach_wait()
    nx, ny, _ = shape
    out = []
    for t in targets:
        if t["status"] != 0 or t["path_offset"] < 0:
            continue
        i = path[t["path_offset"]:t["path_offset"] + t["path_len"]].astype(np.int64)
        cells = np.stack([i % nx, (i // nx) % ny, i // (nx * ny)], 1)
        out.append((cells + np.asarray(origin) + 0.5) * v)
    return out


def initial_points(path, rng, noise):
    """A path thinned to every second voxel, perturbed by `noise` metres, with its start and end repeated three times."""
    keep = path[::2] if len(path) > 2 else path
    keep = np.concatenate([keep, path[-1:]]) if len(path) > 2 and (len(path) - 1) % 2 else keep
    q = keep + rng.standard_normal(keep.shape) * noise
    q[0], q[-1] = path[0], path[-1]
    return np.concatenate([q[:1], q[:1], q, q[-1:], q[-1:]])


def test_drive_fields_equal_the_model():
    """The windowed drive: after every second call a plain or a known field with the signed grid, host copy or
    resident.  The initial trajectories are the voxel-centre paths of a reach job on the latest known field, thinned,
    as they are and with seeded perturbations."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.125
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_signed_enable()
    ctx.trajectory_enable(*CAPS)
    views = Views(ctx, 6)
    ctx.reach_enable(64, 1 << 14, 4096)
    rng = np.random.default_rng(7)
    p = tj.params(1, 10, 1, margin=0.5, v_max=2.0, a_max=4.0, max_iter=40, memory=8, max_ls=10, samples=8, radius=0.25)
    stored, paths, used = set(), [], 0
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = min(T, t0 + 2)
        windowed(ctx, t0, t1, lists, want_counts=False)
        views.capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            ctx.pool_transform(warp(1))
            ctx.inactive_transform(max(stored), warp(2))
            views.warp(warp(1))
        known, host_copy = call % 2 == 1, call % 4 < 2
        c = camera(t1 - 1)
        if known:
            slots, poses = views.request()
            ctx.field_enqueue_known(c, 5, slots, poses, host_copy=host_copy)
            _, origin, _ = ctx.field_wait()
            want = pyoracle_field_known.known_field(field_points(ctx, 5), voxel, shape, c, views.oracle_views(slots), MAX_RANGE)
            sdist = fs.state_field(want[3], voxel)[1]
            found = [q for q in reach_paths(ctx, c, origin, voxel, shape, rng) if 6 <= len(q) <= 480]
            paths = found or paths
        else:
            ctx.field_enqueue(c, 5, host_copy=host_copy)
            _, origin, _ = ctx.field_wait()
            sdist = fs.field(field_points(ctx, 5), voxel, shape, c)[1]
        if not paths:   # no known field yet: lines through the camera positions
            cams = np.array([camera(t)[:3] for t in range(T)], np.float64)
            paths = [a + np.linspace(0, 1, 20)[:, None] * rng.standard_normal(3) * 2 for a in cams[rng.integers(0, T, 4)]]
        else:
            used += 1
        init = [initial_points(q, rng, noise) for q in paths[:8] for noise in (0.0, 0.15)]
        pts = np.concatenate(init)
        ofs = np.concatenate([[0], np.cumsum([len(q) for q in init])]).astype(np.int32)
        equals_the_model(ctx, pts, ofs, rng.uniform(0.2, 1.0, len(init)), p, sdist, origin, voxel,
                         f"call {call} {'known' if known else 'plain'} {'host' if host_copy else 'resident'}")
    assert used > 0, "no reach path to start from"
    ctx.close()


def test_a_job_in_flight_reads_the_old_grid():
    shape, voxel, origin = (32, 32, 16), 0.1, (-16, -16, -8)
    rng = np.random.default_rng(2)
    ctx = known_ctx(shape, voxel)
    grids = crafted_grids(shape, rng)
    ctx.debug_field_load_state(grids["pillar"], origin)
    ctx.field_wait()
    sdist = ctx.field_signed()
    pts, ofs, dt = random_trajectories(rng, origin, voxel, shape, 16)
    p = tj.params(max_iter=30)
    ctx.trajectory_enqueue(pts, ofs, dt, p)
    ctx.debug_field_load_state(grids["random"], (3, 4, 5))    # the next request, before the job's wait
    info, rec, out = ctx.trajectory_wait()
    wq, wr, wi = tj.job(pts, ofs, dt, p, sdist, origin, voxel)
    assert info.tobytes() == wi.tobytes() and rec.tobytes() == wr.tobytes() and out.tobytes() == wq.tobytes()
    ctx.field_wait()
    ctx.close()


@pytest.mark.parametrize("chunk", [1, 4])
def test_trajectory_jobs_change_nothing_else(chunk):
    lists = simple_lists()
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    shape, voxel = (64, 64, 32), 0.1
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.field_signed_enable()
        c.publish_enable()
        c.field_query_enable(512, 4, 64)
    a.trajectory_enable(*CAPS)
    va, vb = Views(a, 4), Views(b, 4)
    rng = np.random.default_rng(chunk)
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c, v in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            v.capture_call(call, t0, t1)
        cam = camera(t1 - 1)
        for c, v in ((a, va), (b, vb)):
            c.field_enqueue_known(cam, 5, *v.request())
        pts, ofs, dt = random_trajectories(rng, (-32, -32, -16), voxel, shape, 4)
        a.trajectory_enqueue(pts, ofs, dt, tj.params(max_iter=20))
        fa, fb = a.field_wait(), b.field_wait()
        a.trajectory_wait()
        assert fa[0].tobytes() == fb[0].tobytes() and a.field_signed().tobytes() == b.field_signed().tobytes()
        q = rng.standard_normal((256, 3))
        res = []
        for c in (a, b):
            c.field_query_enqueue(q, signed=True)
            s = c.field_query_wait()
            c.publish_enqueue(5)
            pu = c.publish_wait()
            res.append([s[0].tobytes(), pu[0].tobytes(), pu[1].tobytes(), pu[2]])
        assert res[0] == res[1], f"call {call}"
        assert map_state(a) == map_state(b), f"call {call}: pool, store or table"
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_the_job():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    a = new_ctx(store=STORE)
    for t0 in range(0, first):
        windowed(a, t0, t0 + 1, lists, want_counts=False)
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    b.field_signed_enable()
    b.trajectory_enable(*CAPS)
    for t0 in range(0, first + 2):
        windowed(b, t0, t0 + 1, lists, want_counts=False)
    c = camera(first - 1)
    b.field_enqueue(c, 1)
    with pytest.raises(capi.DsmError):
        b.field_wait()
    _, ws, o, _ = fs.field(field_points(a, 1), voxel, shape, c)
    rng = np.random.default_rng(5)
    pts, ofs, dt = random_trajectories(rng, o, voxel, shape, 6)
    p = tj.params(max_iter=20)
    b.trajectory_enqueue(pts, ofs, dt, p)
    with pytest.raises(capi.DsmError) as e:
        b.trajectory_wait()
    assert e.value.code == -6
    info, rec, out = e.value.trajectory
    wq, wr, wi = tj.job(pts, ofs, dt, p, ws, o, voxel)
    assert info.tobytes() == wi.tobytes() and rec.tobytes() == wr.tobytes() and out.tobytes() == wq.tobytes()
    a.close()
    b.close()


def test_error_contract():
    lib = capi.load_library()
    P = capi.DsmTrajectoryParams
    pts = np.zeros((8, 3))
    pts[:, 0] = np.arange(8) * 0.1
    ofs = np.array([0, 8], np.int32)
    dt = np.ones(1)
    good = tj.params(memory=4)

    def enq(ctx, p=good, q=pts, o=ofs, d=dt, n=1):
        pp = P(**{k: p[k] for k, _ in P._fields_ if k != "reserved"})
        return lib.dsm_trajectory_enqueue(ctx.h, q.ctypes.data, o.ctypes.data, d.ctypes.data, n, capi.ctypes.byref(pp))

    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    assert lib.dsm_trajectory_enable(None, 1, 8, 1) == -1
    assert lib.dsm_trajectory_enqueue(None, None, None, None, 0, None) == -1
    assert lib.dsm_trajectory_wait(None, None, None, None) == -1
    assert lib.dsm_trajectory_enable(ctx.h, 4, 64, 4) == -7            # before dsm_field_enable
    ctx.field_enable(0.1, 16, 16, 8)
    ctx.views_enable(1, 1.0)
    assert lib.dsm_trajectory_enable(ctx.h, 4, 64, 4) == -7            # before dsm_field_signed_enable
    ctx.field_signed_enable()
    for args in ((0, 64, 4), (4, 0, 4), (4, 64, 0), (4, 64, 17), ((1 << 24) + 1, 64, 4)):
        assert lib.dsm_trajectory_enable(ctx.h, *args) == -1
    assert lib.dsm_trajectory_wait(ctx.h, None, None, None) == -7
    assert lib.dsm_trajectory_enable(ctx.h, 4, 64, 4) == 0
    assert lib.dsm_trajectory_enable(ctx.h, 4, 64, 4) == -7            # once
    assert enq(ctx) == -7                                              # no field request yet
    assert lib.dsm_trajectory_wait(ctx.h, None, None, None) == -7      # nothing enqueued
    st = np.full((8, 16, 16), FREE, np.uint8)
    ctx.debug_field_load_state(st, (-8, -8, -4))
    assert enq(ctx) == 0                                               # the latest request, in flight or not
    assert enq(ctx) == -7                                              # one job in flight
    assert lib.dsm_trajectory_wait(ctx.h, None, None, None) == 0
    ctx.field_wait()
    bad = [dict(p=tj.params(memory=5)), dict(p=tj.params(max_iter=1025)), dict(p=tj.params(max_ls=0)),
           dict(p=tj.params(max_ls=33)), dict(p=tj.params(samples=65)), dict(p=tj.params(samples=0)),
           dict(p=tj.params(radius=-1)), dict(p=tj.params(w_feas=np.inf)), dict(p=tj.params(g_tol=-1)),
           dict(o=np.array([0, 6], np.int32)), dict(o=np.array([1, 8], np.int32)), dict(n=0), dict(n=5),
           dict(d=np.zeros(1)), dict(d=np.full(1, np.nan)), dict(q=np.where(np.arange(24).reshape(8, 3) == 4, np.inf, pts))]
    for kw in bad:
        assert enq(ctx, **kw) == -1, kw
    big = np.zeros((257, 3))
    assert enq(ctx, q=big, o=np.array([0, 257], np.int32)) == -1       # N > 256
    many = np.zeros((70, 3))
    assert enq(ctx, q=many, o=np.array([0, 70], np.int32)) == -1       # more than max_points
    assert enq(ctx, q=np.zeros((16, 3)), o=np.array([0, 8, 7], np.int32), d=np.ones(2), n=2) == -1   # offsets fall
    assert lib.dsm_trajectory_enqueue(ctx.h, None, ofs.ctypes.data, dt.ctypes.data, 1, None) == -1
    ctx.close()
    # the signed grid's pairing rule, and the work bound (2^17 points x 1024 iterations x 33 trials > 2^32)
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 16, 8)
    ctx.views_enable(1, 1.0)
    ctx.debug_field_load_state(np.full((8, 16, 16), FREE, np.uint8), (0, 0, 0))   # without the signed grid
    ctx.field_wait()
    ctx.field_signed_enable()
    ctx.trajectory_enable(512, 1 << 17, 1)
    assert enq(ctx) == -7                                              # the latest request has no signed grid
    ctx.debug_field_load_state(np.full((8, 16, 16), FREE, np.uint8), (0, 0, 0))
    ctx.field_wait()
    n = 512
    q = np.zeros((256 * n, 3))
    q[:, 0] = np.tile(np.arange(256) * 0.01, n)
    o = (np.arange(n + 1) * 256).astype(np.int32)
    heavy = tj.params(max_iter=1024, max_ls=32, memory=1)
    assert enq(ctx, q=q, o=o, d=np.ones(n), n=n, p=heavy) == -1
    assert enq(ctx, q=q, o=o, d=np.ones(n), n=n, p=dict(heavy, max_ls=30)) == 0   # 2^17 x 1024 x 31 < 2^32
    assert lib.dsm_trajectory_wait(ctx.h, None, None, None) == 0
    ctx.close()
    # the bound on final samples: 4 145 trajectories of 256 points at 64 samples per segment pass 2^26
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 16, 8)
    ctx.views_enable(1, 1.0)
    ctx.field_signed_enable()
    n = 4145
    ctx.trajectory_enable(n, 256 * n, 1)
    ctx.debug_field_load_state(np.full((8, 16, 16), FREE, np.uint8), (0, 0, 0))
    ctx.field_wait()
    q = np.zeros((256 * n, 3))
    q[:, 0] = np.tile(np.arange(256) * 0.01, n)
    o = (np.arange(n + 1) * 256).astype(np.int32)
    dense = tj.params(max_iter=0, memory=1, samples=64)
    assert n * (253 * 64 + 1) > tj.MAX_SAMPLES >= (n - 1) * (253 * 64 + 1)
    assert enq(ctx, q=q, o=o, d=np.ones(n), n=n, p=dense) == -1
    assert enq(ctx, q=q, o=o[:n], d=np.ones(n - 1), n=n - 1, p=dense) == 0
    assert lib.dsm_trajectory_wait(ctx.h, None, None, None) == 0
    ctx.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)
RELOAD = 10
PARAMS_DTYPE = np.dtype([(k, "<f8") for k in ("w_smooth", "w_clear", "w_feas", "margin", "v_max", "a_max", "g_tol")] +
                        [(k, "<i4") for k in ("max_iter", "memory", "max_ls", "samples")] + [("radius", "<f4"), ("reserved", "<i4", 3)])


def test_node_trajectories_equal_the_model(tmp_path):
    """The node drive (keyframes, loop closures) through tests/cpp/trajectory_main.cpp: enable_trajectories() refuses
    before enable_signed_distance(), trajectories() before any field and right after load_state; after every fused frame
    its results equal the model on the signed grid, which equals the oracle over the node's own clouds."""
    cam, n = synth.KITTI, 16
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    r = run_driver("trajectory_main", str(tmp_path), cam, sc, [2, 0, 1 << 20, 1 << 21, *FIELD, RELOAD], after=[str(tmp_path / "map")])
    assert r.i() == -7 and r.i() == 0 and r.i() == -7
    pr = r.take(PARAMS_DTYPE, 1)[0]
    p = {k: pr[k].item() for k in tj.PARAM_NAMES}
    moved = 0
    for t in range(n):
        rc, c, origin = r.i(), r.take(np.float64, 3).copy(), r.take(np.int32, 3).copy()
        rs, sdist = r.i(), r.lst(np.float32).reshape(nz, ny, nx)
        rt, pts, ofs, dt = r.i(), r.lst(np.float64).reshape(-1, 3), r.lst(np.int32), r.lst(np.float64)
        info, rec, out = r.take(tj.INFO_DTYPE, 1)[0], r.lst(tj.RECORD_DTYPE), r.lst(np.float64).reshape(-1, 3)
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        assert rc == rs == rt == rr == 0, f"message {t}"
        _, ws, o, _ = fs.field(xyz(act, inact), voxel, (nx, ny, nz), c)
        assert origin.tolist() == o.tolist() and sdist.tobytes() == ws.tobytes(), f"message {t}: signed grid"
        wq, wr, wi = tj.job(pts, ofs, dt, p, sdist, origin, voxel)
        assert info.tobytes() == wi.tobytes() and rec.tobytes() == wr.tobytes() and out.tobytes() == wq.tobytes(), f"message {t}"
        moved += int((out != pts).any())
        if t + 1 == RELOAD:
            assert r.i() == -7, "trajectories() right after load_state"
    assert moved > 0
    assert r.o == len(r.raw)
