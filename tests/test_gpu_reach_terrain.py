"""dsm_reach_enqueue_terrain: driving paths over the latest terrain job's traversable cells, on the device.

The device equals oracle/pyoracle_reach_terrain bit for bit in the whole header (rounds and converged included), the
target records, the path list and the cost grid, on the terrain the device's own terrain job found (which is held to
oracle/pyoracle_terrain first): every known field of the windowed drive with frontier targets (chunks 1 and 4, up -2
and +1), loaded grids for all six up axes, in-plane extents that are not multiples of 32 or 16 and in-plane axes of one
cell, the maze and a serpentine cut short by max_rounds against the round emulator, and a 1024 x 1024 plane converged
against Dijkstra.  A job in flight reads the terrain it was enqueued behind across the next terrain and field requests;
terrain and field jobs alternate on one context, each equal to its own model; a drive with terrain reach jobs leaves
everything as a twin without them.  On the synthetic road (§8.20's request), the model finds a goal ahead on the road
reached over cells at the ground's level, no path entering a box top, and a box top unreachable; the device equals the
model.  The rejected-frame and error contracts, and dsm::SurfelMapNode (tests/cpp/reach_terrain_main.cpp)."""
from functools import partial

import numpy as np
import pytest

import known_space
import pyoracle_frontier
import pyoracle_reach as R
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, NODE_FIELD, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, assert_error_stays, known_drive, node_args,
                         pose12, rejected, rejected_known, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import maze
from resident_map import camera, load_known

pytestmark = pytest.mark.gpu

same = partial(known_space.same, names=("header", "targets", "path list", "cost grid"))
TNAMES = ("info", "level", "status", "step", "clearance")
CAPS, ROUNDS = (64, 1 << 16), 4096


def loader(shape, voxel, up, caps=CAPS, max_rounds=ROUNDS):
    """A context whose field has grid `shape` (nx, ny, nz), with views, terrain (up), frontier and reach jobs enabled."""
    ctx = small_ctx(shape, voxel)
    ctx.terrain_enable(up)
    ctx.frontier_enable(256, 1 << 18)
    ctx.reach_enable(*caps, max_rounds)
    ctx.caps = (caps, max_rounds, up, shape, voxel)
    return ctx


def terrain(ctx, state, origin, headroom=2, max_step=1, what=""):
    """The device's terrain job on the latest known field, held to the model; returns it."""
    _, _, up, _, voxel = ctx.caps
    ctx.terrain_enqueue(headroom, max_step)
    got = ctx.terrain_wait()
    known_space.same(got, TR.job(state, origin, voxel, up, headroom, max_step), f"{what} (terrain)", TNAMES)
    return got


def drive_job(ctx, tr, start, radius, k, goals=(), with_frontiers=False, exact=False, what=""):
    """The device's terrain reach job on terrain tr (the latest terrain job) against the model."""
    (mt, mp), mr, up, shape, voxel = ctx.caps
    fr = None
    if with_frontiers:
        ctx.frontier_enqueue(1)
        fc, fv, _ = ctx.frontier_wait()
        fr = (fc, fv)
    ctx.reach_enqueue_terrain(start, radius, k, goals, with_frontiers, True)
    got = ctx.reach_wait()
    want = RT.job(tr, shape, voxel, start, radius, k, goals, fr, mt, mp, mr, exact)
    same(got, want, what, rounds=not exact)
    return got


def scene(rng, shape, up, p_box=0.06, p_hole=0.03):
    """A state grid [nz][ny][nx]: a flat ground along `up`, boxes three voxels high and holes without support."""
    a = abs(up) - 1
    h0, h1 = RT.plane_axes(up)
    n_a = shape[a]
    g = np.full((shape[h1], shape[h0]), n_a // 3)
    g[rng.random(g.shape) < p_box] += 3
    k = np.arange(n_a)
    up_k = (k if up > 0 else n_a - 1 - k)[None, None, :]
    col = np.where(up_k < g[..., None], UNKNOWN, np.where(up_k == g[..., None], OCCUPIED, FREE)).astype(np.uint8)
    col[rng.random(g.shape) < p_hole] = UNKNOWN
    pos = {h1: 0, h0: 1, a: 2}
    return np.ascontiguousarray(np.transpose(col, (pos[2], pos[1], pos[0])))


def floored(walls, n_up=4):
    """A z-up state grid [n_up][Q][P] whose plane [Q][P] is an occupied floor under free space, and no support at all
    (every voxel unknown) where `walls` holds."""
    Q, P = walls.shape
    st = np.full((n_up, Q, P), FREE, np.uint8)
    st[0] = OCCUPIED
    st[:, walls] = UNKNOWN
    return st


def serpentine_walls(Q, P):
    w = np.zeros((Q, P), bool)
    for i, q in enumerate(range(3, Q - 1, 4)):
        w[q, :] = True
        w[q, P - 1 if i % 2 == 0 else 0] = False
    return w


def point(c, origin, voxel):
    return tuple((c[i] + origin[i] + 0.5) * float(np.float32(voxel)) for i in range(3))


# ---- the windowed drive ----
@pytest.mark.parametrize("chunk,up", [(1, -2), (4, -2), (4, 1)])
def test_drive_known_fields_with_frontier_targets_equal_the_model(chunk, up):
    reached = 0

    def enable(c):
        c.terrain_enable(up)
        c.frontier_enable(256, 1 << 18)
        c.reach_enable(*CAPS, ROUNDS)

    for call, t0, t1, ctx, v, cam, slots, poses, (_, origin, _), state in known_drive((64, 64, 32), chunk, (0.125, 0.1), enable):
        ctx.caps = (CAPS, ROUNDS, up, (64, 64, 32), v)
        tr = terrain(ctx, state, origin, 1 + call % 3, call % 2, f"frames {t0}-{t1 - 1}")
        goals = [tuple(cam + d) for d in ((1.0, 0.0, 1.5), (-1.5, 0.5, 2.5), (0.0, -40.0, 0.0))]
        for radius, k in ((0.0, 2), (v, 4)):
            got = drive_job(ctx, tr, cam, radius, k, goals, True, what=f"frames {t0}-{t1 - 1}, voxel {v}, r {radius}")
            reached += int((got[1]["status"] == 0).sum())
    assert reached > 0 or up != -2   # along +x the drive's columns are mostly without support


# ---- loaded grids ----
@pytest.mark.parametrize("up", TR.UPS)
def test_loaded_grids_equal_the_model(up):
    rng = np.random.default_rng(80 + up)
    shape = [45, 37, 40]
    shape[abs(up) - 1] = 12
    ctx = loader(tuple(shape), 0.1, up)
    for trial in range(3):
        state = scene(rng, shape, up)
        origin = tuple(int(x) for x in rng.integers(-30, 30, 3))
        load_known(ctx, state, origin, 0.1, f"up {up}, trial {trial}")
        tr = terrain(ctx, state, origin, what=f"up {up}")
        for radius, k in ((0.0, 0), (0.1, 1), (0.25, 3)):
            start = point([rng.integers(0, n) for n in shape], origin, 0.1)
            goals = [point([rng.integers(-2, n + 2) for n in shape], origin, 0.1) for _ in range(5)]
            drive_job(ctx, tr, start, radius, k, goals, trial == 2, what=f"up {up}, trial {trial}, r {radius}")
    ctx.close()


@pytest.mark.parametrize("shape,up", [((70, 33, 6), 3), ((97, 5, 49), -2), ((1, 40, 30), -2), ((30, 1, 40), -1), ((45, 8, 1), -2)])
def test_odd_extents_and_one_cell_axes_equal_the_model(shape, up):
    rng = np.random.default_rng(shape[0] * 7 + shape[2])
    ctx = loader(shape, 0.05, up)
    state = scene(rng, list(shape), up, p_box=0.1, p_hole=0.05)
    load_known(ctx, state, (-3, 7, 11), 0.05, str(shape))
    tr = terrain(ctx, state, (-3, 7, 11), what=str(shape))
    for k in (0, 2):
        start = point([rng.integers(0, n) for n in shape], (-3, 7, 11), 0.05)
        goals = [point([rng.integers(0, n) for n in shape], (-3, 7, 11), 0.05) for _ in range(4)]
        drive_job(ctx, tr, start, 0.0, k, goals, k == 2, what=f"{shape}, k {k}")
    ctx.close()


def test_maze_and_serpentine_cut_short_equal_the_emulator():
    """The maze's corridors and a 100 x 48 serpentine, at round caps of 1, 2, 3, 5 and 9, and converged."""
    mz = maze(20, 4)[0] == OCCUPIED
    for name, walls in (("maze", mz), ("serpentine", serpentine_walls(48, 100))):
        st = floored(walls)
        shape = (st.shape[2], st.shape[1], st.shape[0])
        Q, P = walls.shape
        for cap in (1, 2, 3, 5, 9, ROUNDS):
            ctx = loader(shape, 0.1, 3, max_rounds=cap)
            load_known(ctx, st, (0, 0, 0), 0.1, name)
            tr = terrain(ctx, st, (0, 0, 0), what=name)
            goals = [point((p, q, 0), (0, 0, 0), 0.1) for q in range(1, Q, 9) for p in range(1, P, 11)]
            got = drive_job(ctx, tr, point((1, 1, 2), (0, 0, 0), 0.1), 0.0, 1, goals, what=f"{name}, cap {cap}")
            assert got[0]["converged"] == (cap == ROUNDS), (name, cap)
            ctx.close()


def test_a_1024_plane_converges_to_dijkstra():
    rng = np.random.default_rng(11)
    walls = rng.random((1024, 1024)) < 0.08
    walls[:, 300:303] = True
    walls[500:520, 300:303] = False
    st = floored(walls, 3)
    ctx = loader((1024, 1024, 3), 0.1, 3)
    load_known(ctx, st, (0, 0, 0), 0.1, "1024 plane")
    tr = terrain(ctx, st, (0, 0, 0), what="1024 plane")
    goals = [point((1000, 1000, 0), (0, 0, 0), 0.1), point((10, 1010, 0), (0, 0, 0), 0.1), point((700, 20, 2), (0, 0, 0), 0.1)]
    got = drive_job(ctx, tr, point((5, 5, 1), (0, 0, 0), 0.1), 0.0, 2, goals, exact=True, what="1024 plane")
    assert got[0]["converged"] == 1 and (got[1]["status"] == 0).all()
    ctx.close()


# ---- stream order ----
def test_a_job_in_flight_reads_the_terrain_it_was_enqueued_behind():
    """A job enqueued behind a terrain job still in flight, then the next field request and terrain job before its wait,
    reads the first terrain; the next job reads the second."""
    rng = np.random.default_rng(3)
    shape = (50, 12, 40)
    ctx = loader(shape, 0.1, -2)
    a, b = scene(rng, list(shape), -2), scene(rng, list(shape), -2, p_box=0.3)
    load_known(ctx, a, (-5, -5, -5), 0.1, "a")
    start, goals = point((25, 0, 20), (-5, -5, -5), 0.1), [point((3, 0, 38), (-5, -5, -5), 0.1)]
    ctx.terrain_enqueue(2, 1)
    ctx.reach_enqueue_terrain(start, 0.0, 2, goals, False, True)      # behind the terrain job, before its wait
    ctx.debug_field_load_state(b, (3, 4, 5))                           # the next field request
    ta = ctx.terrain_wait()
    known_space.same(ta, TR.job(a, (-5, -5, -5), 0.1, -2, 2, 1), "terrain a", TNAMES)
    ctx.terrain_enqueue(2, 1)                                          # the next terrain job, before the reach wait
    same(ctx.reach_wait(), RT.job(ta, shape, 0.1, start, 0.0, 2, goals, None, *CAPS, ROUNDS), "in flight")
    ctx.field_wait()
    tb = ctx.terrain_wait()
    known_space.same(tb, TR.job(b, (3, 4, 5), 0.1, -2, 2, 1), "terrain b", TNAMES)
    drive_job(ctx, tb, start, 0.0, 2, goals, what="the next terrain")
    ctx.close()


def test_terrain_and_field_jobs_alternate():
    rng = np.random.default_rng(4)
    shape = (40, 10, 36)
    ctx = loader(shape, 0.1, -2)
    state = scene(rng, list(shape), -2)
    dist = load_known(ctx, state, (1, -2, 3), 0.1, "alternate")
    tr = terrain(ctx, state, (1, -2, 3))
    start, goals = point((20, 2, 18), (1, -2, 3), 0.1), [point((2, 2, 30), (1, -2, 3), 0.1), point((39, 8, 1), (1, -2, 3), 0.1)]
    for kind in ("terrain", "field", "field", "terrain", "terrain", "field"):
        if kind == "terrain":
            got = drive_job(ctx, tr, start, 0.0, 2, goals, kind == "terrain", what="terrain")
            assert got[3].shape == (36, 1, 40)
        else:
            ctx.reach_enqueue(start, 0.0, 2, goals, False, True)
            got = ctx.reach_wait()
            same(got, R.reach(state, dist, (1, -2, 3), 0.1, start, 0.0, 2, goals, None, *CAPS, ROUNDS), "field")
            assert got[3].shape == (36, 10, 40)
    ctx.close()


def test_terrain_reach_jobs_change_nothing_else(tmp_path):
    """A drive with terrain and terrain reach jobs beside a publish snapshot and an asynchronous checkpoint leaves the
    map, both published clouds, the fields, the state grids and the checkpoint files byte-identical to a twin without
    them."""
    def enable_a(a):
        a.terrain_enable(-2)
        a.reach_enable(*CAPS, ROUNDS)

    def enqueue(c, is_a, call, t1):
        if is_a:
            c.terrain_enqueue(1 + call % 3, 1)
            c.reach_enqueue_terrain(camera(t1 - 1), 0.0, 2, [tuple(camera(t1 - 1) + (1.0, 0.0, 2.0))], False, True)

    def check(a, outs, call, t1, what):
        state, origin = outs["state"][0], outs["field"][1]
        tr = a.terrain_wait()
        known_space.same(tr, TR.job(state, origin, 0.1, -2, 1 + call % 3, 1), what, TNAMES)
        same(a.reach_wait(), RT.job(tr, (64, 64, 32), 0.1, camera(t1 - 1), 0.0, 2, [tuple(camera(t1 - 1) + (1.0, 0.0, 2.0))], None,
                                    *CAPS, ROUNDS), what)

    twin_drive(tmp_path, lambda c: None, enable_a, enqueue, lambda c: {}, check)


# ---- the synthetic road (DESIGN.md §8.20's request) ----
ROAD_VOXEL, ROAD_SHAPE, ROAD_CENTRE, ROAD_VIEWS = 0.2, (64, 20, 128), (0.0, 1.0, 12.8), 256
BOXES_Z = (5.0, 13.0)


def road_ctx():
    """§8.20's road request: eight KITTI frames, 256 views, a known request at 0.2 m; terrain (up -2) and reach jobs."""
    cam = synth.KITTI
    ctx = capi.Context(cam, max_batch=16, max_local_surfels=1 << 18)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    imgs = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(8)]
    ctx.fuse_stream_resident(list(range(8)), np.stack([g for g, _ in imgs]), np.stack([d for _, d in imgs]),
                             np.stack([synth.pose_stream(t) for t in range(8)]))
    ctx.field_enable(ROAD_VOXEL, *ROAD_SHAPE)
    ctx.views_enable(ROAD_VIEWS, 40.0)
    poses = []
    for j in range(ROAD_VIEWS):
        ctx.views_capture(j % 8, j)
        P = pose12(synth.pose_stream(j % 8))
        P[3] += 0.35 * (j // 8 % 8) - 1.2
        P[11] += 0.8 * (j // 64)
        poses.append(P)
    ctx.field_enqueue_known(ROAD_CENTRE, 1, list(range(ROAD_VIEWS)), np.array(poses))
    _, origin, _ = ctx.field_wait()
    state, _ = ctx.field_state()
    ctx.terrain_enable(-2)
    ctx.reach_enable(*CAPS, ROUNDS)
    ctx.caps = (CAPS, ROUNDS, -2, ROAD_SHAPE, ROAD_VOXEL)
    return ctx, state.copy(), origin.copy()


def test_synthetic_road_semantics():
    """A goal on the road ahead of the first camera is reached over traversable cells at the ground's level and no path
    enters a box top; a goal on the first box's top, which no supported cell neighbours at its level, is not reached at
    approach 0.  Asserted on the model, then the device equals the model."""
    ctx, state, origin = road_ctx()
    v = float(np.float32(ROAD_VOXEL))
    ground = int(np.floor(1.65 / v)) - origin[1]
    top = int(np.floor(0.65 / v)) - origin[1]
    tr = TR.job(state, origin, ROAD_VOXEL, -2, 5, 1)
    L, S = tr[1][:, 0, :], tr[2][:, 0, :]                     # [z][x]
    xs = (np.arange(ROAD_SHAPE[0]) + origin[0] + 0.5) * v
    zs = (np.arange(ROAD_SHAPE[2]) + origin[2] + 0.5) * v
    box = np.argwhere((L == top) & (np.abs(zs - BOXES_Z[0])[:, None] <= 1.0) & (np.abs(xs - 2.5)[None, :] <= 1.0))
    assert len(box) > 0
    bz, bx = box[0]
    # the start and the goal: the traversable road cells nearest the middle of the road 8 m and 11 m ahead
    road = np.argwhere((S == FREE) & (L == ground) & (np.abs(xs) <= 1.0)[None, :])
    near = [road[np.argmin(np.abs(zs[road[:, 0]] - z) + np.abs(xs[road[:, 1]]))] for z in (8.0, 11.0)]
    start, ahead = [(xs[x], 1.6, zs[z]) for z, x in near]
    goals = [ahead, (xs[bx], 0.65, zs[bz])]
    info, recs, path, cost = RT.job(tr, ROAD_SHAPE, ROAD_VOXEL, start, 0.0, 2, goals[:1])
    assert info["start_status"] == 0 and info["converged"] == 1
    assert recs[0]["status"] == 0, recs
    P = ROAD_SHAPE[0]
    seg = path[recs[0]["path_offset"]:recs[0]["path_offset"] + recs[0]["path_len"]]
    assert (S.reshape(-1)[seg] == FREE).all() and (L.reshape(-1)[seg] == ground).all()
    assert not (L.reshape(-1)[path] == top).any()
    rec_box = RT.job(tr, ROAD_SHAPE, ROAD_VOXEL, start, 0.0, 0, goals[1:])[1][0]
    assert (rec_box["status"], rec_box["target"]) == (2, bz * P + bx)
    got_tr = terrain(ctx, state, origin, 5, 1, "road")
    drive_job(ctx, got_tr, start, 0.0, 2, goals[:1], what="road")
    drive_job(ctx, got_tr, start, 0.0, 0, goals[1:], what="road box")
    ctx.close()


# ---- the rejected frame and the error contract ----
def test_rejected_frame_comes_back_from_wait():
    def enqueue(b, first):
        b.terrain_enqueue(3, 1)
        b.reach_enqueue_terrain(camera(first - 1), 0.0, 2, [tuple(camera(first - 1) + (1.0, 0.0, 1.0))], False, True)

    r = rejected_known(lambda b: (b.terrain_enable(-2), b.reach_enable(*CAPS, ROUNDS)), enqueue)
    e = rejected(r.ctx.reach_wait)
    tr = rejected(r.ctx.terrain_wait).terrain
    known_space.same(tr, TR.job(r.state, r.field[1], r.voxel, -2, 3, 1), "rejected terrain", TNAMES)
    same(e.reach, RT.job(tr, r.shape, r.voxel, camera(r.first - 1), 0.0, 2, [tuple(camera(r.first - 1) + (1.0, 0.0, 1.0))], None,
                         *CAPS, ROUNDS), "rejected")
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    st3 = (capi.ctypes.c_double * 3)(0.05, 0.05, 0.05)
    enq = lambda c, radius=0.0, k=0, goals=None, n=0, fr=0: lib.dsm_reach_enqueue_terrain(c, st3, radius, k, goals, n, fr, 0)
    assert enq(None) == -1
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 12, 8)
    ctx.views_enable(1, 1.0)
    ctx.terrain_enable(3)
    assert enq(ctx.h) == -7                                  # before dsm_reach_enable
    ctx.reach_enable(4, 64, 64)
    ctx.frontier_enable(16, 1024)
    assert enq(ctx.h) == -7                                  # no terrain job yet
    st = np.full((8, 12, 16), FREE, np.uint8)
    st[0] = OCCUPIED
    st[:, :, 15] = UNKNOWN
    ctx.debug_field_load_state(st, (0, 0, 0))
    ctx.field_wait()
    ctx.frontier_enqueue(1)                                  # on this request
    ctx.frontier_wait()
    ctx.terrain_enqueue(2, 0)                                # in flight: a job may run behind it
    g = np.zeros((5, 3))
    for kw in (dict(radius=float("nan")), dict(radius=-1.0), dict(radius=float("inf")), dict(k=-1), dict(k=5),
               dict(goals=g.ctypes.data, n=5), dict(n=1), dict(n=-1)):
        assert enq(ctx.h, **kw) == -1, kw
    bad = np.array([[0.0, float("nan"), 0.0]])
    assert enq(ctx.h, goals=bad.ctypes.data, n=1) == -1
    assert lib.dsm_reach_enqueue_terrain(ctx.h, None, 0.0, 0, None, 0, 0, 0) == -1
    assert enq(ctx.h, fr=1) == 0                             # the frontier job read the terrain job's request
    assert enq(ctx.h) == -7                                  # one reach job in flight
    assert lib.dsm_reach_enqueue(ctx.h, st3, 0.0, 0, None, 0, 0, 0) == -7
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == 0
    ctx.terrain_wait()
    ctx.debug_field_load_state(st, (0, 0, 0))                # a later field request: the terrain job stays the latest
    ctx.field_wait()
    assert enq(ctx.h, fr=1) == 0                             # the frontier and terrain jobs read the same older request
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == 0
    ctx.frontier_enqueue(1)                                  # a frontier job on the newer request
    ctx.frontier_wait()
    assert enq(ctx.h, fr=1) == -7
    assert enq(ctx.h) == 0
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == 0
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == -7
    ctx.close()


# ---- the node ----
def test_node_reach_terrain_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, terrain(), frontiers() and
    reach_terrain(with_frontiers) from the field's middle equal the model over the grid the driver dumps; clouds, PLY
    and PCD files equal a twin without these jobs; reach_terrain() before terrain() on the frame, with frontiers before
    frontiers(), and after load_state until the next fused frame returns DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("reach_terrain_main", str(tmp_path), cam, sc, node_args() + [64, 1 << 16, 2048, RELOAD], tag="a", after=[pa])
    q = run_driver("reach_terrain_main", str(tmp_path), cam, sc, node_args() + [0, 0, 0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, k = r.i(), r.i()
        start = r.take(np.float64, 3).copy()
        radius = float(r.take(np.float32, 1)[0])
        goal = r.take(np.float64, 3).copy()
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        info = r.take(np.uint8, R.INFO_DTYPE.itemsize).view(R.INFO_DTYPE)[0].copy()
        targets, path = r.lst(R.TARGET_DTYPE), r.lst(np.int32)
        before_terrain, before_frontiers, after_load = r.i(), r.i(), r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        tr = TR.job(state, origin, voxel, -2, 3, 1)
        want = RT.job(tr, (nx, ny, nz), voxel, start, radius, k, [goal], (clusters, vox), 64, 1 << 16, 2048)
        same((info, targets, path, None), want, f"message {t}")
        found += int((targets["status"] == 0).sum()) > 0
        assert before_terrain == -7 and before_frontiers == -7, f"message {t}"
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: reach_terrain() after load_state"
    assert found > 0
    twin_node_tail(r, q, pa, pb)
