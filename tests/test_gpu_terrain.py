"""dsm_terrain_enable / _enqueue / _wait: where a ground robot can drive on the known field, on the device.

Every level, status, step and clearance, the counts and the origin equal oracle/pyoracle_terrain bit for bit on the
windowed drive's known fields (chunks 1 and 4, with loop-closure warps between calls) and on loaded grids: random grids
at three densities for all six up axes, an up axis of 1024 voxels, 1024 x 1024 cells under a short up axis, an in-plane
axis of one voxel, the maze and the serpentine.  On the synthetic road seen by the KITTI camera, the model (asserted
first, on the device's own state grid) finds the road ahead of the first camera traversable at the ground's level and
the box tops at box height, blocked where they meet supported road.  A job in flight across the next field request
reads the old grid; a drive with terrain jobs leaves the map, the fields, the state
grids, the published clouds and the checkpoint files byte-identical to a twin's without them.  The rejected-frame and
error contracts, and dsm::SurfelMapNode (tests/cpp/terrain_main.cpp)."""
import numpy as np
import pytest

import pyoracle_terrain as TR
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, NODE_FIELD, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, assert_error_stays, known_drive, node_args,
                         rejected, rejected_known, same, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import maze, serpentine
from known_space import pose12
from resident_map import load_known

pytestmark = pytest.mark.gpu

NAMES = ("info", "level", "status", "step", "clearance")


def device_equals_model(ctx, state, origin, voxel, up, headroom, max_step, what):
    ctx.terrain_enqueue(headroom, max_step)
    got = ctx.terrain_wait()
    same(got, TR.job(state, origin, voxel, up, headroom, max_step), what, NAMES)
    return got


@pytest.mark.parametrize("chunk,up", [(1, -2), (4, -2), (4, 1)])
def test_drive_known_fields_equal_the_model(chunk, up):
    """The windowed drive with warps between calls: after every call, terrain jobs on the known field at the camera at
    two headrooms and two step limits."""
    traversable = 0
    for call, t0, t1, ctx, v, cam, slots, poses, (_, origin, _), state in known_drive((64, 64, 32), chunk, (0.125, 0.1),
                                                                                     lambda c: c.terrain_enable(up)):
        for headroom, max_step in ((1 + call % 3, call % 2), (6, 3)):
            got = device_equals_model(ctx, state, origin, v, up, headroom, max_step, f"frames {t0}-{t1 - 1}, voxel {v}, h {headroom}")
            traversable += int(got[0]["n_traversable"])
    assert traversable > 0


# ---- the synthetic road (DESIGN.md §8.20) ----
# Eight KITTI frames of synth.py's drive fused once; each frame's rays captured into 32 of 256 view slots, the views
# moved across the road in eight steps of 0.35 m and along it in four of 0.8 m, as a drive's keyframes overlap.  A known
# request at 0.2 m on a 64 x 20 x 128 grid centred 1 m below and 12.8 m ahead of the first camera (x -6.4..6.4 m,
# y -1.2..2.8 m, z -0.2..25.4 m), every fused surfel; up = -2, headroom 5 voxels (1 m), max_step 1.
ROAD_VOXEL, ROAD_SHAPE, ROAD_CENTRE, ROAD_VIEWS = 0.2, (64, 20, 128), (0.0, 1.0, 12.8), 256
ROAD_HEADROOM, ROAD_STEP = 5, 1
BOXES_Z = (5.0, 13.0)   # the front panels of synth.py's boxes: z = 8k + 5, |x - 2.5| < 1 m, y 0.65..1.65 m


def road_state():
    """The state grid and origin of the road request, from the device."""
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
    return ctx, state.copy(), origin.copy()


def test_synthetic_road_semantics():
    """The road ahead of the first camera (|x| <= 1 m, z 8..11 m) is supported at the ground's voxel (y = 1.65 m) and
    mostly traversable, at 1 m of headroom and at the 1.8 m of INTEGRATION.md's example.  Each box's front panel is
    supported at the box's top voxel (y = 0.65 m); where its top meets supported road, the 1 m step blocks it.  Asserted
    on the model over the device's state grid, then the device equals the model."""
    ctx, state, origin = road_state()
    v = float(np.float32(ROAD_VOXEL))
    xs = (np.arange(ROAD_SHAPE[0]) + origin[0] + 0.5) * v
    zs = (np.arange(ROAD_SHAPE[2]) + origin[2] + 0.5) * v
    ground = int(np.floor(1.65 / v)) - origin[1]
    top = int(np.floor(0.65 / v)) - origin[1]
    road = np.ix_(np.flatnonzero((zs >= 8.0) & (zs <= 11.0)), [0], np.flatnonzero(np.abs(xs) <= 1.0))
    for headroom in (ROAD_HEADROOM, 9):
        info, lev, status, step, clear = TR.job(state, origin, ROAD_VOXEL, -2, headroom, ROAD_STEP)
        rl, rs = lev[road], status[road]
        assert (rl[rl >= 0] == ground).all(), (headroom, np.unique(rl, return_counts=True))
        assert (rs == FREE).mean() >= 0.75, (headroom, np.unique(rs, return_counts=True))
    info, lev, status, step, clear = TR.job(state, origin, ROAD_VOXEL, -2, ROAD_HEADROOM, ROAD_STEP)
    h = TR.height(lev[road], origin, ROAD_VOXEL, -2)
    assert np.allclose(h[np.isfinite(h)], -1.6)          # the top face of the ground's voxel, 1.6 m below y = 0
    L, S = lev[:, 0, :], status[:, 0, :]
    edges = 0
    for zf in BOXES_Z:
        panel = np.ix_(np.flatnonzero(np.abs(zs - zf) <= v), np.flatnonzero(np.abs(xs - 2.5) <= 0.8))
        pl = L[panel]
        assert ((pl == -1) | ((pl >= top) & (pl < ground))).all(), (zf, np.unique(pl, return_counts=True))
        assert (pl == top).sum() >= 0.75 * (pl >= 0).sum() and (pl == top).sum() >= 8, (zf, np.unique(pl, return_counts=True))
        assert np.allclose(TR.height(pl[pl == top], origin, ROAD_VOXEL, -2), -0.6)
    near = (np.abs(zs - np.array(BOXES_Z)[:, None]) <= v).any(axis=0)[:, None] & (np.abs(xs - 2.5) <= 1.0)[None, :]
    for zi, xi in zip(*np.nonzero(near & (L >= top) & (L < ground))):
        nb = L[max(zi - 1, 0):zi + 2, max(xi - 1, 0):xi + 2]
        if (nb == ground).any():                          # a box top beside supported road: a step of 4 voxels or more
            assert S[zi, xi] == OCCUPIED, (zs[zi], xs[xi])
            edges += 1
    assert edges >= 8, edges
    device_equals_model(ctx, state, origin, ROAD_VOXEL, -2, ROAD_HEADROOM, ROAD_STEP, "synthetic road")
    ctx.close()


# ---- loaded grids ----
def random_grid(rng, shape, density):
    """Independent random states per voxel: occupied with probability 0.7 density, unknown 0.3 density, else free."""
    nx, ny, nz = shape
    st = rng.choice(np.array([FREE, OCCUPIED, UNKNOWN], np.uint8), size=(nz, ny, nx), p=(1 - density, density * 0.7, density * 0.3))
    return st


def columns_grid(rng, shape, up):
    """A terrain along `up`: a rolling ground with steps of 0..3 voxels between neighbours, free above, unknown below."""
    nx, ny, nz = shape
    a = abs(up) - 1
    n_a = shape[a]
    hor = [k for k in range(3) if k != a]
    g = np.cumsum(rng.integers(-1, 2, size=(shape[hor[1]], shape[hor[0]])), axis=1) + n_a // 3
    g = np.clip(g + rng.integers(0, 2, size=g.shape) * rng.integers(0, 4, size=g.shape), 0, n_a - 2)
    k = np.arange(n_a)
    ground = g[..., None]                                     # [h1][h0][k], k the coordinate along a
    up_k = k[None, None, :] if up > 0 else (n_a - 1 - k)[None, None, :]
    up_g = ground if up > 0 else n_a - 1 - ground
    col = np.where(up_k < up_g, UNKNOWN, np.where(up_k == up_g, OCCUPIED, FREE)).astype(np.uint8)
    # [h1][h0][a] -> [z][y][x]
    order = {2: (2, 0, 1), 1: (0, 2, 1), 0: (0, 1, 2)}[a]
    return np.ascontiguousarray(np.transpose(col, order))


SHAPE = (37, 29, 13)


@pytest.mark.parametrize("up", TR.UPS)
def test_loaded_random_grids_equal_the_model(up):
    rng = np.random.default_rng(40 + up)
    ctx = small_ctx(SHAPE, 0.1)
    ctx.terrain_enable(up)
    n_a = SHAPE[abs(up) - 1]
    for density in (0.05, 0.3, 0.7):
        state = random_grid(rng, SHAPE, density)
        origin = tuple(int(x) for x in rng.integers(-50, 50, 3))
        load_known(ctx, state, origin, 0.1, f"density {density}")
        for headroom, max_step in ((1, 0), (2, 1), (n_a - 1, 1023)):
            device_equals_model(ctx, state, origin, 0.1, up, headroom, max_step, f"up {up}, density {density}, h {headroom}")
    state = columns_grid(rng, SHAPE, up)
    load_known(ctx, state, (0, 0, 0), 0.1, "columns")
    for max_step in (0, 1, 2):
        got = device_equals_model(ctx, state, (0, 0, 0), 0.1, up, 3, max_step, f"up {up}, columns, step {max_step}")
        assert got[0]["n_support"] > 0
    ctx.close()


@pytest.mark.parametrize("shape,up", [((8, 1024, 6), -2), ((3, 5, 1024), 3), ((1024, 1024, 4), 3), ((1, 40, 30), -2),
                                      ((1, 40, 30), 3), ((30, 1, 40), -1)])
def test_loaded_grids_at_the_limits_equal_the_model(shape, up):
    """An up axis of 1024 voxels, 1024 x 1024 cells under a short up axis, and in-plane axes of one voxel."""
    rng = np.random.default_rng(shape[0] + abs(up))
    ctx = small_ctx(shape, 0.05)
    ctx.terrain_enable(up)
    state = columns_grid(rng, shape, up)
    load_known(ctx, state, (-3, 7, 11), 0.05, str(shape))
    n_a = shape[abs(up) - 1]
    for headroom, max_step in ((1, 1), (min(3, n_a - 1), 0), (n_a - 1, 2)):
        device_equals_model(ctx, state, (-3, 7, 11), 0.05, up, headroom, max_step, f"{shape}, h {headroom}")
    noisy = random_grid(rng, shape, 0.2)
    load_known(ctx, noisy, (0, 0, 0), 0.05, f"{shape} random")
    device_equals_model(ctx, noisy, (0, 0, 0), 0.05, up, 1, 0, f"{shape} random")
    ctx.close()


def test_maze_and_serpentine_equal_the_model():
    """The maze on an occupied floor (corridors traversable, walls without support) and the serpentine."""
    st = maze(12, 3)
    floored = np.concatenate([np.full((1,) + st.shape[1:], OCCUPIED, np.uint8), st])   # z up: floor, then two layers
    shape = (floored.shape[2], floored.shape[1], floored.shape[0])
    ctx = small_ctx(shape, 0.1)
    ctx.terrain_enable(3)
    load_known(ctx, floored, (0, 0, 0), 0.1, "maze")
    got = device_equals_model(ctx, floored, (0, 0, 0), 0.1, 3, 2, 0, "maze")
    assert got[0]["n_traversable"] == (st[0] == FREE).sum() and got[0]["n_blocked"] == 0
    ctx.close()
    sp = serpentine(20, 9, 7)
    ctx = small_ctx((20, 9, 7), 0.1)
    ctx.terrain_enable(-2)
    sp = sp.copy()
    sp[sp == UNKNOWN] = OCCUPIED
    load_known(ctx, sp, (1, 2, 3), 0.1, "serpentine")
    for headroom in (1, 2):
        device_equals_model(ctx, sp, (1, 2, 3), 0.1, -2, headroom, 1, f"serpentine h {headroom}")
    ctx.close()


def test_a_job_in_flight_reads_the_old_grid():
    rng = np.random.default_rng(2)
    ctx = small_ctx(SHAPE, 0.1)
    ctx.terrain_enable(-2)
    a, b = columns_grid(rng, SHAPE, -2), random_grid(rng, SHAPE, 0.3)
    load_known(ctx, a, (-5, -5, -5), 0.1, "a")
    ctx.terrain_enqueue(3, 1)
    ctx.debug_field_load_state(b, (3, 4, 5))    # the next request, before the job's wait
    same(ctx.terrain_wait(), TR.job(a, (-5, -5, -5), 0.1, -2, 3, 1), "in flight", NAMES)
    ctx.field_wait()
    device_equals_model(ctx, b, (3, 4, 5), 0.1, -2, 3, 1, "the next grid")
    ctx.close()


def test_terrain_jobs_change_nothing_else(tmp_path):
    """A drive with terrain jobs beside a publish snapshot and an asynchronous checkpoint leaves the map, both published
    clouds, the fields, the state grids and the checkpoint files byte-identical to a twin without them."""
    def enqueue(c, is_a, call, t1):
        if is_a:
            c.terrain_enqueue(1 + call % 4, call % 3)

    def check(a, outs, call, t1, what):
        same(a.terrain_wait(), TR.job(outs["state"][0], outs["field"][1], 0.1, -2, 1 + call % 4, call % 3), what, NAMES)

    twin_drive(tmp_path, lambda c: None, lambda a: a.terrain_enable(-2), enqueue, lambda c: {}, check)


def test_rejected_frame_comes_back_from_wait():
    r = rejected_known(lambda b: b.terrain_enable(-2), lambda b, first: b.terrain_enqueue(3, 1))
    e = rejected(r.ctx.terrain_wait)
    same(e.terrain, TR.job(r.state, r.field[1], r.voxel, -2, 3, 1), "rejected", NAMES)
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    assert lib.dsm_terrain_enable(None, 3) == -1
    assert lib.dsm_terrain_enqueue(None, 1, 0) == -1
    assert lib.dsm_terrain_wait(None, None, None, None, None, None) == -1
    assert lib.dsm_terrain_enable(ctx.h, 3) == -7                     # before dsm_field_enable
    ctx.field_enable(0.1, 16, 12, 8)
    assert lib.dsm_terrain_enable(ctx.h, 3) == -7                     # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert lib.dsm_terrain_enqueue(ctx.h, 1, 0) == -7                 # before dsm_terrain_enable
    assert lib.dsm_terrain_wait(ctx.h, None, None, None, None, None) == -7
    for up in (0, 4, -4, 100):
        assert lib.dsm_terrain_enable(ctx.h, up) == -1
    assert lib.dsm_terrain_enable(ctx.h, 3) == 0
    assert lib.dsm_terrain_enable(ctx.h, 3) == -7                     # once
    assert lib.dsm_terrain_enqueue(ctx.h, 1, 0) == -7                 # no field request yet
    ctx.field_enqueue((0, 0, 0), 1)                                   # a plain field request: not a known one
    ctx.field_wait()
    assert lib.dsm_terrain_enqueue(ctx.h, 1, 0) == -7
    st = np.full((8, 12, 16), FREE, np.uint8)
    st[0] = OCCUPIED
    ctx.debug_field_load_state(st, (0, 0, 0))
    for headroom, max_step in ((0, 0), (8, 0), (-1, 0), (1, -1), (1, 1024)):   # n_z = 8: headroom in [1, 7]
        assert lib.dsm_terrain_enqueue(ctx.h, headroom, max_step) == -1, (headroom, max_step)
    assert lib.dsm_terrain_enqueue(ctx.h, 7, 1023) == 0               # the latest request, in flight or not
    assert lib.dsm_terrain_enqueue(ctx.h, 7, 1023) == -7              # one job in flight
    assert lib.dsm_terrain_wait(ctx.h, None, None, None, None, None) == 0
    assert lib.dsm_terrain_wait(ctx.h, None, None, None, None, None) == -7   # nothing in flight
    ctx.field_wait()
    device_equals_model(ctx, st, (0, 0, 0), 0.1, 3, 7, 0, "the whole column free")
    ctx.close()


# ---- the node ----
def test_node_terrain_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, terrain() equals the model over the grid the
    driver dumps; clouds, PLY and PCD files equal a twin without terrain jobs; enable_terrain() before
    enable_known_space, terrain() before any field and right after load_state return DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("terrain_main", str(tmp_path), cam, sc, node_args() + [1, RELOAD], tag="a", after=[pa])
    q = run_driver("terrain_main", str(tmp_path), cam, sc, node_args() + [0, RELOAD], tag="b", after=[pb])
    assert r.i() == -7 and r.i() == 0 and r.i() == -7
    supported = 0
    for t in range(n):
        rc, headroom, max_step = r.i(), r.i(), r.i()
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        info = r.take(np.uint8, TR.INFO_DTYPE.itemsize).view(TR.INFO_DTYPE)[0].copy()
        m = TR.terrain_shape((nx, ny, nz), -2)
        planes = (r.lst(np.int16), r.lst(np.uint8), r.lst(np.uint8), r.lst(np.float32))
        after_load = r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        got = (info,) + tuple(p.reshape(m[2], m[1], m[0]) for p in planes)
        same(got, TR.job(state, origin, voxel, -2, headroom, max_step), f"message {t}", NAMES)
        supported += int(info["n_support"])
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: terrain() after load_state"
    assert supported > 0
    twin_node_tail(r, q, pa, pb)
