"""dsm_viewpoint_enqueue_terrain: viewpoints of a ground robot, candidate cells of the latest terrain job's plane around
each frontier cluster, each camera eye voxels above its cell's support and scored through the known field, on the
device.

The device equals oracle/pyoracle_viewpoint_terrain bit for bit in the header, every record and every slot, on the
terrain the device's own terrain job found (itself held to oracle/pyoracle_terrain): every known field of the windowed
drive (chunks 1 and 4, up -2 and +1, with and without reach, both blocking rules, 8 and 64 rotations), loaded grids for
all six up axes, in-plane extents that are not multiples of 32 or 16 and one-cell axes, and a sampling cut.  Each
returned viewpoint of a fully sampled cluster, re-scored by a gain job at its camera pose naming its cluster, gives
n_cluster == n_seen; with reach each cost is the host-copy cost plane of the terrain reach job.  Stream order across the
next field request, terrain, frontier and reach jobs, the pairing refusals, field and terrain viewpoint jobs
alternating, a drive with terrain viewpoint jobs against a twin without them, the rejected frame, every error code, the
node (tests/cpp/viewpoint_terrain_main.cpp), and the whole ground chain on the synthetic road: terrain, frontiers, a
terrain reach job with frontiers, the terrain viewpoints with reach, the matrix over the robot and the chosen cameras,
and the tour."""
import ctypes
from functools import partial

import numpy as np
import pytest

import known_space
import pyoracle_frontier
import pyoracle_gain as G
import pyoracle_reach as R
import pyoracle_reach_matrix_terrain as RMT
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR
import pyoracle_tour as TM
import pyoracle_viewpoint as V
import pyoracle_viewpoint_terrain as VT
import road_scene
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from ground_views import WIDE, rotations, scene
from known_space import (FREE, K, NODE_FIELD, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, assert_error_stays, gcam, known_drive, node_args,
                         rejected, rejected_known, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import params
from resident_map import load_known

pytestmark = pytest.mark.gpu

INF = V.INF
ROUNDS = 4096
same = partial(known_space.same, names=("header", "clusters", "viewpoints"))
TNAMES = ("info", "level", "status", "step", "clearance")


def field_tiles(shape):
    return int(np.prod([(n + 7) // 8 for n in shape]))


def rot_tables(up):
    """8 rotations (four headings level, two pitched up and down) and 64 (16 headings at four pitches)."""
    return np.concatenate([rotations(up, 4), rotations(up, 2, (0.35, -0.35))]), rotations(up, 16, (0.0, 0.3, -0.3, 0.6))


def loader(shape, voxel, up, gain=256):
    ctx = small_ctx(shape, voxel)
    ctx.terrain_enable(up)
    ctx.frontier_enable(256, 1 << 18)
    ctx.reach_enable(16, 1 << 12, ROUNDS)
    ctx.gain_enable(gain)
    ctx.viewpoint_enable(64, 1 << 18)
    return ctx


def terrain(ctx, state, origin, voxel, up, headroom, max_step=1, what=""):
    """The device's terrain job on the latest known field, held to the model; returns it."""
    ctx.terrain_enqueue(headroom, max_step)
    got = ctx.terrain_wait()
    known_space.same(got, TR.job(state, origin, voxel, up, headroom, max_step), f"{what} (terrain)", TNAMES)
    return got


def rescore(ctx, got, fr, cam, rot, tr, voxel, eye):
    """Every returned viewpoint of a cluster whose members are all samples, scored by a gain job at its camera pose
    naming its cluster: n_cluster == n_seen."""
    _, recs, slots = got
    poses, cl, want = [], [], []
    for i, r in enumerate(recs):
        if r["status"] != 0 or r["n_samples"] != fr[0][r["cluster"]]["n_voxels"]:
            continue
        for s in slots[i]:
            if s["voxel"] >= 0:
                t = VT.camera_point(int(s["voxel"]), tr, voxel, eye)
                poses.append(np.concatenate([rot[s["rotation"]].reshape(3, 3), t[:, None]], axis=1).reshape(12))
                cl.append(r["cluster"])
                want.append(s["n_seen"])
    if not poses:
        return 0
    ctx.gain_enqueue(cam, poses, np.array(cl, np.int32))
    _, g = ctx.gain_wait()
    assert g["n_cluster"].tolist() == want
    return len(poses)


def vjob(ctx, state, voxel, tr, fr, cam, rot, cl, prm, eye, cost=None, what=""):
    """The device's terrain viewpoint job against the model, re-scored by gain jobs; with reach, every cost is the cost
    plane's."""
    ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, eye)
    got = ctx.viewpoint_wait()
    same(got, VT.viewpoints(state, voxel, tr, cam, rot, cl, prm, eye, fr, cost), what)
    rescore(ctx, got, fr, cam, rot, tr, voxel, eye)
    if prm.with_reach:
        s = got[2][got[2]["voxel"] >= 0]
        assert (s["cost"] == cost.reshape(-1)[s["voxel"]]).all() and (s["cost"] != INF).all(), what
    return got


def frontiers(ctx, m=1):
    ctx.frontier_enqueue(m)
    fc, fv, _ = ctx.frontier_wait()
    return fc, fv


def reach_plane(ctx, start, radius=0.0):
    ctx.reach_enqueue_terrain(start, radius, 2, None, False, True)
    return ctx.reach_wait()[3]


def ring_start(tr, voxel, rng):
    """A world point at the centre of a random traversable cell of terrain tr (any height)."""
    up = int(tr[0]["up"])
    h0, h1 = RT.plane_axes(up)
    cells = np.flatnonzero(tr[2].reshape(-1) == FREE)
    c = int(rng.choice(cells))
    P = int(tr[0]["m"][h0])
    p = [0.0, 0.0, 0.0]
    v = float(np.float32(voxel))
    p[h0], p[h1] = (int(tr[0]["origin"][h0]) + c % P + 0.5) * v, (int(tr[0]["origin"][h1]) + c // P + 0.5) * v
    return tuple(p)


# ---- the windowed drive ----
@pytest.mark.parametrize("chunk,up", [(1, -2), (4, -2), (4, 1)])
def test_drive_known_fields_equal_the_model(chunk, up):
    shape = (64, 64, 32)
    rot8, rot64 = rot_tables(up)
    found = 0

    def enable(c):
        c.terrain_enable(up)
        c.frontier_enable(256, 1 << 18)
        c.reach_enable(16, 1 << 12, ROUNDS)
        c.gain_enable(2048)
        c.viewpoint_enable(64, 1 << 18)

    for call, t0, t1, ctx, v, cam, slots, poses, (_, origin, _), state in known_drive(shape, chunk, (0.125, 0.1), enable):
        what = f"frames {t0}-{t1 - 1}, voxel {v}"
        headroom = 2 + call % 2
        tr = terrain(ctx, state, origin, v, up, headroom, call % 2, what)
        fr = frontiers(ctx, 1 + call % 2)
        with_reach, ub = call % 2, (call // 2) % 2
        cost = reach_plane(ctx, cam) if with_reach else None
        rot = rot64 if call % 3 == 2 else rot8
        gc = gcam(K, (10 + 7 * (call % 3)) * np.float32(v), ub)
        prm = params(1 + call % 2, 5, 0, 1 + call % 2, top_k=1 + 5 * (call % 4), with_reach=with_reach)
        cl = (np.arange(min(len(fr[0]) + 2, 12)) if len(fr[0]) else np.array([0, 3])).astype(np.int32)
        got = vjob(ctx, state, v, tr, fr, gc, rot, cl, prm, 1 + call % headroom, cost, what)
        found += int(got[1]["n_viewpoints"].sum())
    assert found > 0 or up != -2


# ---- loaded grids ----
@pytest.mark.parametrize("up", TR.UPS)
def test_loaded_grids_equal_the_model(up):
    rng = np.random.default_rng(220 + up)
    shape = [45, 37, 40]
    shape[abs(up) - 1] = 12
    ctx = loader(tuple(shape), 0.1, up)
    rot8, rot64 = rot_tables(up)
    for trial in range(2):
        state = scene(rng, shape, up, p_box=0.06, p_hole=0.04)
        origin = tuple(int(x) for x in rng.integers(-30, 30, 3))
        load_known(ctx, state, origin, 0.1, f"up {up}, trial {trial}")
        tr = terrain(ctx, state, origin, 0.1, up, 3, what=f"up {up}")
        fr = frontiers(ctx)
        cl = np.arange(min(len(fr[0]), 16))
        cost = reach_plane(ctx, ring_start(tr, 0.1, rng))
        for ub, rot, eye, prm in [(0, rot8, 1, params(1, 6, 0, 1, top_k=8)), (1, rot64, 3, params(2, 8, 0, 2, top_k=4, with_reach=1)),
                                  (1, rot8, 2, params(0, 4, 0, 1, top_k=16, radius=0.1, with_reach=1))]:
            vjob(ctx, state, 0.1, tr, fr, gcam(K, 1.2, ub), rot, cl, prm, eye, cost if prm.with_reach else None,
                 f"up {up}, trial {trial}, eye {eye}")
    ctx.close()


@pytest.mark.parametrize("shape,up", [((70, 33, 6), 3), ((97, 5, 49), -2), ((1, 40, 30), -2), ((30, 1, 40), -1), ((45, 8, 1), -2)])
def test_odd_extents_and_one_cell_axes_equal_the_model(shape, up):
    rng = np.random.default_rng(shape[0] * 7 + shape[2])
    ctx = loader(shape, 0.05, up)
    state = scene(rng, list(shape), up, p_box=0.1, p_hole=0.08)
    load_known(ctx, state, (-3, 7, 11), 0.05, str(shape))
    tr = terrain(ctx, state, (-3, 7, 11), 0.05, up, 2, what=str(shape))
    fr = frontiers(ctx)
    cl = np.append(np.arange(min(len(fr[0]), 40)), len(fr[0]))     # and one past the table
    rot8, _ = rot_tables(up)
    for ub, eye in ((0, 1), (1, 2)):
        vjob(ctx, state, 0.05, tr, fr, gcam(K, 0.6, ub), rot8, cl, params(0, 5, 0, 1, top_k=6), eye, what=f"{shape}, eye {eye}")
    ctx.close()


def test_sampling_cut():
    """A floor whose far row is a frontier wall of 40 x 7 voxels: n_samples is min(max_samples, 280)."""
    shape, voxel = (40, 36, 8), 0.2
    st = np.full(shape[::-1], FREE, np.uint8)
    st[0] = OCCUPIED
    st[1:, 30:, :] = UNKNOWN
    ctx = loader(shape, voxel, 3)
    load_known(ctx, st, (0, 0, 0), voxel, "cut")
    tr = terrain(ctx, st, (0, 0, 0), voxel, 3, 4, what="cut")
    fr = frontiers(ctx)
    assert len(fr[0]) == 1
    for ms in (1, 7, 100, 4096):
        got = vjob(ctx, st, voxel, tr, fr, WIDE._replace(max_range=4.0), rotations(3, 8), [0], params(0, 10, 0, 2, top_k=6, max_samples=ms),
                   2, what=f"cut {ms}")
        assert got[1][0]["n_samples"] == min(ms, int(fr[0][0]["n_voxels"])) and got[1][0]["n_viewpoints"] > 0
    ctx.close()


# ---- stream order and pairing ----
def test_stream_order_and_pairing():
    """A job reads the field, terrain, frontier and reach results it was enqueued behind, not the next ones; it needs the
    latest field request to be the terrain job's, a frontier job on it, and with reach a terrain reach job on the latest
    terrain job."""
    rng = np.random.default_rng(9)
    shape, voxel, up = (50, 12, 40), 0.1, -2
    ctx = loader(shape, voxel, up)
    a, b = scene(rng, list(shape), up), scene(rng, list(shape), up, p_box=0.2)
    oa, ob = (-5, -5, -5), (3, 4, 5)
    rot, _ = rot_tables(up)
    cam = gcam(K, 1.5, 1)
    prm = params(1, 6, 0, 1, top_k=4, with_reach=1)
    cl = np.arange(8)
    ta_model = TR.job(a, oa, voxel, up, 2, 1)
    start = ring_start(ta_model, voxel, rng)
    ctx.debug_field_load_state(a, oa)
    ctx.terrain_enqueue(2, 1)
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)            # no frontier job on this field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)            # with reach, no reach job on this terrain
    assert e.value.code == -7
    ctx.reach_enqueue_terrain(start, 0.0, 1, None, False, True)
    ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)                # before the field, terrain, frontier and reach waits
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)            # one job in flight
    assert e.value.code == -7
    ctx.field_wait()
    ta, fra, ra = ctx.terrain_wait(), ctx.frontier_wait(), ctx.reach_wait()
    known_space.same(ta, ta_model, "terrain a", TNAMES)
    want = VT.viewpoints(a, voxel, ta, cam, rot, cl, prm, 2, fra[:2], ra[3])
    ctx.debug_field_load_state(b, ob)                                  # the next field request, terrain, frontier and reach jobs
    ctx.terrain_enqueue(2, 1)
    ctx.frontier_enqueue(1)
    ctx.reach_enqueue_terrain(start, 0.0, 1, None, False, True)
    same(ctx.viewpoint_wait(), want, "in flight")
    ctx.field_wait()
    tb, frb, rb = ctx.terrain_wait(), ctx.frontier_wait(), ctx.reach_wait()
    known_space.same(tb, TR.job(b, ob, voxel, up, 2, 1), "terrain b", TNAMES)
    vjob(ctx, b, voxel, tb, frb[:2], cam, rot, cl, prm, 2, rb[3], "the next terrain")
    # a second terrain job on the same field request: the reach job ran on the first one
    ctx.terrain_enqueue(3, 1)
    tb3 = ctx.terrain_wait()
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)
    assert e.value.code == -7
    vjob(ctx, b, voxel, tb3, frb[:2], cam, rot, cl, prm._replace(with_reach=0), 3, what="headroom 3, no reach")
    rb3 = reach_plane(ctx, start)
    vjob(ctx, b, voxel, tb3, frb[:2], cam, rot, cl, prm, 3, rb3, "headroom 3, reach")
    ctx.reach_enqueue(start, 0.0, 1, None, False, False)               # a field reach job
    ctx.reach_wait()
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, 2)
    assert e.value.code == -7
    ctx.debug_field_load_state(a, oa)                                  # a field request the terrain job did not read
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm._replace(with_reach=0), 2)
    assert e.value.code == -7
    ctx.field_wait()
    ctx.terrain_enqueue(2, 1)                                          # a terrain job on it, the frontier job still on b
    with pytest.raises(capi.DsmError) as e:
        ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm._replace(with_reach=0), 2)
    assert e.value.code == -7
    ctx.terrain_wait()
    ctx.close()


def test_field_and_terrain_jobs_alternate():
    rng = np.random.default_rng(4)
    shape, voxel, up = (40, 10, 36), 0.1, -2
    ctx = loader(shape, voxel, up)
    state = scene(rng, list(shape), up)
    dist = load_known(ctx, state, (1, -2, 3), voxel, "alternate")
    tr = terrain(ctx, state, (1, -2, 3), voxel, up, 2)
    fr = frontiers(ctx)
    rot, _ = rot_tables(up)
    cam = gcam(K, 1.5, 0)
    cl = np.arange(min(len(fr[0]), 8))
    for kind in ("terrain", "field", "field", "terrain", "terrain", "field"):
        if kind == "terrain":
            vjob(ctx, state, voxel, tr, fr, cam, rot, cl, params(1, 5, 0, 1, top_k=4), 2, what="terrain")
        else:
            prm = params(1, 4, 1, 1, top_k=4)
            ctx.viewpoint_enqueue(cam, rot, cl, prm)
            same(ctx.viewpoint_wait(), V.viewpoints(state, dist, (1, -2, 3), voxel, cam, rot, cl, prm, fr), "field")
    ctx.close()


def test_terrain_viewpoint_jobs_change_nothing_else(tmp_path):
    rot, _ = rot_tables(-2)
    cam = gcam(K, 1.5, 1)
    prm = params(1, 5, 0, 1, top_k=3)

    def enable_a(a):
        a.terrain_enable(-2)
        a.frontier_enable(64, 1 << 16)
        a.viewpoint_enable(8, 1 << 14)

    def enqueue(c, is_a, call, t1):
        if is_a:
            c.terrain_enqueue(2 + call % 2, 1)
            c.frontier_enqueue(1)
            c.viewpoint_enqueue_terrain(cam, rot, np.arange(4), prm, 1 + call % 2)

    def check(a, outs, call, t1, what):
        state, origin = outs["state"][0], outs["field"][1]
        tr = a.terrain_wait()
        known_space.same(tr, TR.job(state, origin, 0.1, -2, 2 + call % 2, 1), what, TNAMES)
        fr = a.frontier_wait()
        same(a.viewpoint_wait(), VT.viewpoints(state, 0.1, tr, cam, rot, np.arange(4), prm, 1 + call % 2, fr[:2]), what)

    twin_drive(tmp_path, lambda c: None, enable_a, enqueue, lambda c: {}, check)


# ---- the ground chain on the synthetic road ----
def test_ground_chain_on_the_synthetic_road():
    """terrain(5, 1), frontiers, a terrain reach job with frontiers from the road 8 m ahead, terrain viewpoints with reach
    at eye 4 (0.7 m above the road), the matrix over the start and the chosen cameras, then the tour: asserted on the
    model, then the device equals the model."""
    ctx, state, origin = road_scene.road_request()
    voxel, shape = road_scene.ROAD_VOXEL, road_scene.ROAD_SHAPE
    v = float(np.float32(voxel))
    up, eye = -2, 4
    ctx.terrain_enable(up)
    ctx.frontier_enable(256, 1 << 18)
    ctx.reach_enable(255, 1 << 16, ROUNDS)
    ctx.viewpoint_enable(256, 1 << 20)
    ctx.gain_enable(1024)
    ctx.reach_matrix_enable(256, field_tiles(shape), ROUNDS)
    ctx.tour_enable(256, 4)
    tr = terrain(ctx, state, origin, voxel, up, 5, 1, "road")
    L, S = tr[1][:, 0, :], tr[2][:, 0, :]
    ground = int(np.floor(1.65 / v)) - origin[1]
    xs = (np.arange(shape[0]) + origin[0] + 0.5) * v
    zs = (np.arange(shape[2]) + origin[2] + 0.5) * v
    road = np.argwhere((S == FREE) & (L == ground) & (np.abs(xs) <= 1.0)[None, :])
    z, x = road[np.argmin(np.abs(zs[road[:, 0]] - 8.0) + np.abs(xs[road[:, 1]]))]
    start = (xs[x], 1.6, zs[z])
    fc, fv = frontiers(ctx)
    ctx.reach_enqueue_terrain(start, 0.0, 2, None, True, True)
    rgot = ctx.reach_wait()
    known_space.same(rgot, RT.job(tr, shape, voxel, start, 0.0, 2, (), (fc, fv), 255, 1 << 16, ROUNDS), "road reach",
                     ("header", "targets", "path list", "cost grid"))
    cost = rgot[3]
    rot = rotations(up, 8, (0.0, -0.3))
    cam = gcam(K, 12.0, 1)
    cl = np.arange(min(len(fc), 64))
    prm = params(0, 8, 0, 2, max_samples=256, top_k=1, with_reach=1)
    want = VT.viewpoints(state, voxel, tr, cam, rot, cl, prm, eye, (fc, fv), cost)
    # the model: every viewpoint is a traversable, reached cell whose camera voxel is free, eye voxels above the road
    slots = want[2][:, 0]
    slots = slots[slots["voxel"] >= 0]
    assert len(slots) > 2
    P = shape[0]
    for s in slots:
        c = int(s["voxel"])
        assert S.reshape(-1)[c] == FREE and cost.reshape(-1)[c] == s["cost"] != R.INF
        k = VT.camera_voxel(c % P, c // P, L, up, eye)
        assert state[k[2], k[1], k[0]] == FREE and L.reshape(-1)[c] - k[1] == eye
    pts = [start] + [tuple(VT.camera_point(int(s["voxel"]), tr, voxel, eye)) for s in slots]
    info, sites, M = RMT.matrix(tr, voxel, pts, 0.0, 2, field_tiles(shape), ROUNDS, 256)
    assert (sites["status"] == 0).all() and (sites["approach"] == 0).all() and (sites["voxel"][1:] == slots["voxel"]).all()
    assert (M[0, 1:].astype(np.int64) == slots["cost"].astype(np.int64)).all()   # the same start cell, both converged
    tinfo, starts, order = TM.tour(M, 1, 4, 16, 7)
    assert tinfo["n_included"] == len(pts) and tinfo["n_infinite"] == 0
    # the device
    ctx.viewpoint_enqueue_terrain(cam, rot, cl, prm, eye)
    got = ctx.viewpoint_wait()
    same(got, want, "road viewpoints")
    rescore(ctx, got, (fc, fv), cam, rot, tr, voxel, eye)
    ctx.reach_matrix_enqueue_terrain(pts, 0.0, 2)
    mgot = ctx.reach_matrix_wait()
    known_space.same(mgot, (info, sites, M), "road matrix", ("header", "sites", "matrix"))
    ctx.tour_enqueue(mgot[2], 1, 4, 16, 7)
    known_space.same(ctx.tour_wait(), (tinfo, starts, order), "road tour", ("header", "starts", "order"))
    ctx.close()


# ---- the rejected frame and the error contract ----
def test_rejected_frame_comes_back_from_wait():
    rot, _ = rot_tables(-2)
    cam = gcam(K, 1.5, 1)
    prm = params(1, 5, 0, 1, top_k=3)

    def enqueue(b, first):
        b.terrain_enqueue(3, 1)
        b.frontier_enqueue(1)
        b.viewpoint_enqueue_terrain(cam, rot, np.arange(6), prm, 2)

    r = rejected_known(lambda b: (b.terrain_enable(-2), b.frontier_enable(64, 1 << 16), b.viewpoint_enable(8, 1 << 14)), enqueue)
    e = rejected(r.ctx.viewpoint_wait)
    tr = rejected(r.ctx.terrain_wait).terrain
    known_space.same(tr, TR.job(r.state, r.field[1], r.voxel, -2, 3, 1), "rejected terrain", TNAMES)
    fr = rejected(r.ctx.frontier_wait).frontier
    same(e.viewpoint, VT.viewpoints(r.state, r.voxel, tr, cam, rot, np.arange(6), prm, 2, fr[:2]), "rejected")
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    cam = capi.DsmGainCamera(4.0, 4.0, 3.5, 3.5, 8, 8, 1.0, 1)
    R8 = np.ascontiguousarray(rotations(3, 8))
    cl = np.zeros(2, np.int32)
    ok = capi.DsmViewpointParams(1, 3, 0, 1, 64, 0, 2, 0, 0.0, 0)

    def enq(c, camera=ctypes.byref(cam), rot=R8.ctypes.data, n_rot=8, clusters=cl.ctypes.data, n=2, prm=ok, eye=1):
        return lib.dsm_viewpoint_enqueue_terrain(c, camera, rot, n_rot, clusters, n, None if prm is None else ctypes.byref(prm), eye)

    assert enq(None) == -1
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 12, 8)
    ctx.views_enable(1, 1.0)
    ctx.terrain_enable(3)
    ctx.frontier_enable(64, 1 << 12)
    ctx.reach_enable(4, 1 << 10, 64)
    assert enq(ctx.h) == -7                                  # before dsm_viewpoint_enable
    ctx.viewpoint_enable(4, 1 << 12)
    assert enq(ctx.h) == -7                                  # no terrain job yet
    st = np.full((8, 12, 16), FREE, np.uint8)
    st[0] = OCCUPIED
    st[1:, 10:, :] = UNKNOWN
    ctx.debug_field_load_state(st, (0, 0, 0))
    ctx.field_wait()
    assert enq(ctx.h) == -7                                  # a field request is no terrain job
    ctx.terrain_enqueue(3, 0)                                # in flight: a job may run behind it
    assert enq(ctx.h) == -7                                  # no frontier job on that request
    ctx.frontier_enqueue(1)
    bad = [dict(camera=None), dict(rot=None), dict(n_rot=0), dict(n_rot=65), dict(clusters=None), dict(n=-1), dict(n=5), dict(prm=None),
           dict(eye=0), dict(eye=4), dict(eye=-3), dict(camera=ctypes.byref(capi.DsmGainCamera(0.0, 4.0, 3.5, 3.5, 8, 8, 1.0, 1)))]
    for p in (capi.DsmViewpointParams(1, 3, 1, 1, 64, 0, 2, 0, 0.0, 0), capi.DsmViewpointParams(1, 3, 0, 1, 64, 0, 17, 0, 0.0, 0),
              capi.DsmViewpointParams(1, 3, 0, 0, 64, 0, 2, 0, 0.0, 0), capi.DsmViewpointParams(1, 3, 0, 1, 64, 0, 2, 2, 0.0, 0),
              capi.DsmViewpointParams(1, 3, 0, 1, 64, 0, 2, 0, float("nan"), 0), capi.DsmViewpointParams(0, 40, 0, 1, 64, 0, 2, 0, 0.0, 0)):
        bad.append(dict(prm=p))
    for kw in bad:
        assert enq(ctx.h, **kw) == -1, kw
    wr = capi.DsmViewpointParams(1, 3, 0, 1, 64, 0, 2, 1, 0.0, 0)
    assert enq(ctx.h, prm=wr) == -7                          # with reach, no reach job
    ctx.reach_enqueue((0.55, 0.55, 0.15), 0.0, 1, None, False, False)
    assert enq(ctx.h, prm=wr) == -7                          # a field reach job
    ctx.reach_wait()
    ctx.reach_enqueue_terrain((0.55, 0.55, 0.15), 0.0, 1, None, False, False)
    assert enq(ctx.h, prm=wr, eye=3) == 0                    # eye = headroom, behind the terrain reach job
    assert enq(ctx.h) == -7                                  # one viewpoint job in flight
    assert lib.dsm_viewpoint_enqueue(ctx.h, ctypes.byref(cam), R8.ctypes.data, 8, cl.ctypes.data, 2, ctypes.byref(ok)) == -7
    assert lib.dsm_viewpoint_wait(ctx.h, None, None, None) == 0
    assert lib.dsm_viewpoint_wait(ctx.h, None, None, None) == -7
    ctx.terrain_wait()
    ctx.frontier_wait()
    ctx.reach_wait()
    ctx.close()


# ---- the node ----
def test_node_viewpoints_terrain_equal_the_model_and_change_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, terrain(3, 1), frontiers(), reach_terrain()
    from the field's middle and viewpoints_terrain() over every cluster, with reach on every other frame, equal the
    model over the grid, frontiers, start and rotations the driver dumps; clouds, PLY and PCD files equal a twin without
    these jobs; viewpoints_terrain() before terrain() on the frame and after load_state until the next fused frame
    returns DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("viewpoint_terrain_main", str(tmp_path), cam, sc, node_args() + [1, RELOAD], tag="a", after=[pa])
    q = run_driver("viewpoint_terrain_main", str(tmp_path), cam, sc, node_args() + [0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, ub = r.i(), r.i()
        max_range = float(r.take(np.float32, 1)[0])
        eye = r.i()
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        start = r.take(np.float64, 3).copy()
        rot = r.lst(np.float64).reshape(-1, 9)
        named = r.lst(np.int32)
        prm = V.Params(*r.take(np.int32, 8).tolist(), float(r.take(np.float32, 1)[0]))
        info = r.take(np.uint8, V.INFO_DTYPE.itemsize).view(V.INFO_DTYPE)[0].copy()
        recs = r.lst(V.CLUSTER_DTYPE)
        slots = r.lst(V.VIEWPOINT_DTYPE).reshape(len(recs), -1)
        before_terrain, after_load = r.i(), r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        tr = TR.job(state, origin, voxel, -2, 3, 1)
        gc = G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, max_range, ub)
        cost = None
        if prm.with_reach:
            cost = RT.job(tr, (nx, ny, nz), voxel, tuple(start), prm.radius, 1, max_targets=8, max_path=1 << 12, max_rounds=ROUNDS)[3]
        same((info, recs, slots), VT.viewpoints(state, voxel, tr, gc, rot, named, prm, eye, (clusters, vox), cost), f"message {t}")
        found += int((recs["n_viewpoints"] > 0).sum()) > 0
        assert before_terrain == -7, f"message {t}"
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: viewpoints_terrain() after load_state"
    assert found > 0
    twin_node_tail(r, q, pa, pb)
