"""dsm_reach_matrix_enqueue_terrain: driving costs between many sites over the latest terrain job's traversable cells, on
the device.

The device equals oracle/pyoracle_reach_matrix_terrain bit for bit in the header, the site records and the matrix, on
the terrain the device's own terrain job found (itself held to oracle/pyoracle_terrain): every known field of the
windowed drive (chunks 1 and 4, up -2 and +1; sites the camera, a terrain reach job's viewpoints and random points),
loaded grids for all six up axes, odd in-plane extents and one-cell axes, a density sweep at n_points = max_sites, the
maze and a serpentine cut short at 1, 7 and 40 rounds, and a 1024 x 1024 plane converged against Dijkstra.  Row i equals
the host-copy cost grid of a dsm_reach_enqueue_terrain job from site i, converged and at 7 rounds.  Both sides of the
capacity cut on the flat tile count, a job in flight across the next field request and terrain job, terrain and field
matrix jobs alternating, a drive with terrain matrix jobs against a twin without them, the rejected frame, every error
code, the node (tests/cpp/reach_matrix_terrain_main.cpp), and the whole ground chain on the synthetic road: terrain,
frontiers, a terrain reach job with frontiers, the matrix over the start and the viewpoint cells, and the tour."""
from functools import partial

import numpy as np
import pytest

import known_space
import pyoracle_reach as R
import pyoracle_reach_matrix as RM
import pyoracle_reach_matrix_terrain as RMT
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR
import pyoracle_tour as TM
import road_scene
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, NODE_FIELD, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, assert_error_stays, known_drive, node_args,
                         rejected, rejected_known, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import maze
from resident_map import camera, load_known

pytestmark = pytest.mark.gpu

same = partial(known_space.same, names=("header", "sites", "matrix"))
TNAMES = ("info", "level", "status", "step", "clearance")
ROUNDS = 4096


def field_tiles(shape):
    return int(np.prod([(n + 7) // 8 for n in shape]))


def loader(shape, voxel, up, max_sites=64, max_tiles=None, max_rounds=ROUNDS, reach=None):
    """A context whose field has grid `shape` (nx, ny, nz), with views, terrain (up) and matrix jobs enabled (max_tiles:
    the field's tile count, the most enable takes), and reach jobs with `reach` = (max_targets, max_path) capacities."""
    ctx = small_ctx(shape, voxel)
    ctx.terrain_enable(up)
    mt = field_tiles(shape) if max_tiles is None else max_tiles
    ctx.reach_matrix_enable(max_sites, mt, max_rounds)
    if reach:
        ctx.reach_enable(*reach, max_rounds)
    ctx.mcaps = (mt, max_rounds, max_sites, up, shape, voxel)
    return ctx


def terrain(ctx, state, origin, headroom=2, max_step=1, what=""):
    """The device's terrain job on the latest known field, held to the model; returns it."""
    up, voxel = ctx.mcaps[3], ctx.mcaps[5]
    ctx.terrain_enqueue(headroom, max_step)
    got = ctx.terrain_wait()
    known_space.same(got, TR.job(state, origin, voxel, up, headroom, max_step), f"{what} (terrain)", TNAMES)
    return got


def mjob(ctx, tr, points, radius, k, exact=False, what=""):
    """The device's terrain matrix job on terrain tr (the latest terrain job) against the model.  exact: the model's rows
    are Dijkstra's, every site must be converged, and rounds are not compared."""
    mt, mr, ms, _, _, voxel = ctx.mcaps
    ctx.reach_matrix_enqueue_terrain(points, radius, k)
    got = ctx.reach_matrix_wait()
    want = RMT.matrix(tr, voxel, points, radius, k, mt, mr, ms, exact)
    if exact:
        info, sites = got[0].copy(), got[1].copy()
        assert (sites["converged"] == 1).all(), f"{what}: not converged"
        info["rounds"] = want[0]["rounds"]
        ok = sites["voxel"] >= 0
        sites["rounds"][ok], sites["converged"][ok] = -1, -1
        got = (info, sites, got[2])
    same(got, want, what)
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
    """A z-up state grid [n_up][Q][P]: an occupied floor under free space, and no support where `walls` holds."""
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


def cell_centres(cells, tr, voxel, height):
    """World points at the centres of plane cells q P + p of terrain tr, at `height` along the up axis."""
    up = int(tr[0]["up"])
    h0, h1 = RT.plane_axes(up)
    P = int(tr[0]["m"][h0])
    v = float(np.float32(voxel))
    out = []
    for c in np.asarray(cells).tolist():
        p = [float(height)] * 3
        p[h0] = (int(tr[0]["origin"][h0]) + c % P + 0.5) * v
        p[h1] = (int(tr[0]["origin"][h1]) + c // P + 0.5) * v
        out.append(tuple(p))
    return out


def random_points(rng, shape, origin, voxel, n, pad=2):
    return [point([rng.integers(-pad, s + pad) for s in shape], origin, voxel) for _ in range(n)]


# ---- the windowed drive ----
@pytest.mark.parametrize("chunk,up", [(1, -2), (4, -2), (4, 1)])
def test_drive_known_fields_equal_the_model(chunk, up):
    shape = (64, 64, 32)
    rng = np.random.default_rng(chunk * 10 + up)
    finite = 0

    def enable(c):
        c.terrain_enable(up)
        c.frontier_enable(256, 1 << 18)
        c.reach_enable(31, 1 << 16, ROUNDS)
        c.reach_matrix_enable(64, field_tiles(shape), ROUNDS)

    for call, t0, t1, ctx, v, cam, slots, poses, (_, origin, _), state in known_drive(shape, chunk, (0.125, 0.1), enable):
        ctx.mcaps = (field_tiles(shape), ROUNDS, 64, up, shape, v)
        what = f"frames {t0}-{t1 - 1}, voxel {v}"
        tr = terrain(ctx, state, origin, 1 + call % 3, call % 2, what)
        ctx.frontier_enqueue(1)
        ctx.frontier_wait()
        ctx.reach_enqueue_terrain(cam, 0.0, 2, None, True)
        rinfo, recs, _, _ = ctx.reach_wait()
        vps = recs["viewpoint"][recs["status"] == 0]
        pts = [tuple(cam)] + cell_centres(vps, tr, v, cam[abs(up) - 1]) + random_points(rng, shape, origin, v, 6)
        for radius, k in ((0.0, 2), (v, 4)):
            got = mjob(ctx, tr, pts[:64], radius, k, what=f"{what}, r {radius}")
            finite += int((got[2] != R.INF).sum()) > len(got[1])
    assert finite > 0 or up != -2


# ---- loaded grids ----
@pytest.mark.parametrize("up", TR.UPS)
def test_loaded_grids_equal_the_model(up):
    rng = np.random.default_rng(120 + up)
    shape = [45, 37, 40]
    shape[abs(up) - 1] = 12
    ctx = loader(tuple(shape), 0.1, up)
    for trial in range(2):
        state = scene(rng, shape, up)
        origin = tuple(int(x) for x in rng.integers(-30, 30, 3))
        load_known(ctx, state, origin, 0.1, f"up {up}, trial {trial}")
        tr = terrain(ctx, state, origin, what=f"up {up}")
        trav = RMT.plane(tr, 0.0)[0]
        cells = rng.choice(np.flatnonzero(trav), size=8, replace=False)
        pts = cell_centres(cells, tr, 0.1, rng.uniform(-9, 9)) + random_points(rng, shape, origin, 0.1, 8)
        for radius, k in ((0.0, 0), (0.1, 1), (0.25, 3)):
            mjob(ctx, tr, pts, radius, k, what=f"up {up}, trial {trial}, r {radius}")
    ctx.close()


@pytest.mark.parametrize("shape,up", [((70, 33, 6), 3), ((97, 5, 49), -2), ((1, 40, 30), -2), ((30, 1, 40), -1), ((45, 8, 1), -2)])
def test_odd_extents_and_one_cell_axes_equal_the_model(shape, up):
    rng = np.random.default_rng(shape[0] * 7 + shape[2])
    ctx = loader(shape, 0.05, up)
    state = scene(rng, list(shape), up, p_box=0.1, p_hole=0.05)
    load_known(ctx, state, (-3, 7, 11), 0.05, str(shape))
    tr = terrain(ctx, state, (-3, 7, 11), what=str(shape))
    for k in (0, 2):
        mjob(ctx, tr, random_points(rng, shape, (-3, 7, 11), 0.05, 10, pad=1), 0.0, k, what=f"{shape}, k {k}")
    ctx.close()


def test_density_sweep_at_max_sites():
    rng = np.random.default_rng(21)
    Q, P = 64, 96
    ctx = loader((P, Q, 4), 0.1, 3, max_sites=128)
    for p_wall in (0.02, 0.15, 0.35):
        st = floored(rng.random((Q, P)) < p_wall)
        load_known(ctx, st, (2, -5, 0), 0.1, f"density {p_wall}")
        tr = terrain(ctx, st, (2, -5, 0), what=f"density {p_wall}")
        pts = random_points(rng, (P, Q, 4), (2, -5, 0), 0.1, 128, pad=0)
        got = mjob(ctx, tr, pts, 0.0, 1, what=f"density {p_wall}")
        assert got[0]["n_sites"] == 128
    ctx.close()


def test_maze_and_serpentine_cut_short_equal_the_emulator():
    mz = maze(20, 4)[0] == OCCUPIED
    for name, walls in (("maze", mz), ("serpentine", serpentine_walls(48, 100))):
        st = floored(walls)
        shape = (st.shape[2], st.shape[1], st.shape[0])
        Q, P = walls.shape
        pts = [point((p, q, 2), (0, 0, 0), 0.1) for q in range(1, Q, 9) for p in range(1, P, 11)]
        for cap in (1, 7, 40):
            ctx = loader(shape, 0.1, 3, max_rounds=cap)
            load_known(ctx, st, (0, 0, 0), 0.1, name)
            tr = terrain(ctx, st, (0, 0, 0), what=name)
            got = mjob(ctx, tr, pts, 0.0, 1, what=f"{name}, cap {cap}")
            assert cap > 7 or (got[1]["converged"][got[1]["status"] == 0] == 0).any(), (name, cap)
            ctx.close()


def test_a_1024_plane_converges_to_dijkstra():
    rng = np.random.default_rng(11)
    walls = rng.random((1024, 1024)) < 0.08
    walls[:, 300:303] = True
    walls[500:520, 300:303] = False
    st = floored(walls, 3)
    ctx = loader((1024, 1024, 3), 0.1, 3, max_sites=16, max_tiles=2048)
    load_known(ctx, st, (0, 0, 0), 0.1, "1024 plane")
    tr = terrain(ctx, st, (0, 0, 0), what="1024 plane")
    pts = [point((5, 5, 1), (0, 0, 0), 0.1), point((1000, 1000, 0), (0, 0, 0), 0.1)] + random_points(rng, (1024, 1024, 3), (0, 0, 0), 0.1,
                                                                                                       14, pad=0)
    got = mjob(ctx, tr, pts, 0.0, 2, exact=True, what="1024 plane")
    assert got[0]["n_active_tiles"] == 2048 and (got[2][0] != R.INF).sum() > 8
    ctx.close()


# ---- rows are terrain reach jobs ----
def test_rows_equal_terrain_reach_jobs_from_each_site():
    """Row i equals the host-copy cost grid of a dsm_reach_enqueue_terrain job from site i, read at the sites, with that
    job's start, rounds, converged and reached count; converged and cut at 7 rounds."""
    rng = np.random.default_rng(8)
    walls = serpentine_walls(48, 100) | (rng.random((48, 100)) < 0.05)
    st = floored(walls)
    shape = (100, 48, 4)
    for cap in (7, ROUNDS):
        ctx = loader(shape, 0.1, 3, max_rounds=cap, reach=(4, 1 << 12))
        load_known(ctx, st, (1, 2, 3), 0.1, "rows")
        tr = terrain(ctx, st, (1, 2, 3), what="rows")
        pts = random_points(rng, shape, (1, 2, 3), 0.1, 12, pad=0)
        info, sites, M = mjob(ctx, tr, pts, 0.0, 2, what=f"rows, cap {cap}")
        u = sites["voxel"]
        for i, p in enumerate(pts):
            ctx.reach_enqueue_terrain(p, 0.0, 2, None, False, True)
            rinfo, _, _, cost = ctx.reach_wait()
            assert rinfo["start_voxel"] == u[i] and rinfo["start_status"] == sites[i]["status"]
            assert (rinfo["rounds"], rinfo["converged"], rinfo["n_reached"]) == \
                (sites[i]["rounds"], sites[i]["converged"], sites[i]["n_reached"]), i
            flat = cost.reshape(-1)
            want = np.where((u >= 0) & (u[i] >= 0), flat[np.maximum(u, 0)], R.INF).astype(np.uint32)
            assert M[i].tobytes() == want.tobytes(), i
        assert cap == ROUNDS or (sites["converged"][u >= 0] == 0).any()
        ctx.close()


# ---- the capacity cut ----
def test_both_sides_of_the_capacity_cut():
    rng = np.random.default_rng(5)
    st = floored(rng.random((40, 90)) < 0.3)
    shape = (90, 40, 4)
    n_active = 3 * 3
    pts = random_points(rng, shape, (0, 0, 0), 0.1, 6, pad=0)
    for mt in (n_active, n_active - 1):
        ctx = loader(shape, 0.1, 3, max_tiles=mt)
        load_known(ctx, st, (0, 0, 0), 0.1, "cut")
        tr = terrain(ctx, st, (0, 0, 0), what="cut")
        info = mjob(ctx, tr, pts, 0.0, 1, what=f"max_tiles {mt}")[0]
        assert info["n_active_tiles"] == n_active and info["status"] == int(mt < n_active)
        ctx.close()


# ---- stream order ----
def test_a_job_in_flight_reads_the_terrain_it_was_enqueued_behind():
    rng = np.random.default_rng(3)
    shape = (50, 12, 40)
    ctx = loader(shape, 0.1, -2)
    a, b = scene(rng, list(shape), -2), scene(rng, list(shape), -2, p_box=0.3)
    load_known(ctx, a, (-5, -5, -5), 0.1, "a")
    pts = random_points(rng, shape, (-5, -5, -5), 0.1, 10, pad=0)
    ctx.terrain_enqueue(2, 1)
    ctx.reach_matrix_enqueue_terrain(pts, 0.0, 2)      # behind the terrain job, before its wait
    ctx.debug_field_load_state(b, (3, 4, 5))           # the next field request
    ta = ctx.terrain_wait()
    known_space.same(ta, TR.job(a, (-5, -5, -5), 0.1, -2, 2, 1), "terrain a", TNAMES)
    ctx.terrain_enqueue(2, 1)                          # the next terrain job, before the matrix wait
    same(ctx.reach_matrix_wait(), RMT.matrix(ta, 0.1, pts, 0.0, 2, field_tiles(shape), ROUNDS), "in flight")
    ctx.field_wait()
    tb = ctx.terrain_wait()
    known_space.same(tb, TR.job(b, (3, 4, 5), 0.1, -2, 2, 1), "terrain b", TNAMES)
    mjob(ctx, tb, pts, 0.0, 2, what="the next terrain")
    ctx.close()


def test_terrain_and_field_jobs_alternate():
    rng = np.random.default_rng(4)
    shape = (40, 10, 36)
    ctx = loader(shape, 0.1, -2)
    state = scene(rng, list(shape), -2)
    dist = load_known(ctx, state, (1, -2, 3), 0.1, "alternate")
    tr = terrain(ctx, state, (1, -2, 3))
    pts = random_points(rng, shape, (1, -2, 3), 0.1, 9, pad=0)
    for kind in ("terrain", "field", "field", "terrain", "terrain", "field"):
        if kind == "terrain":
            mjob(ctx, tr, pts, 0.0, 2, what="terrain")
        else:
            ctx.reach_matrix_enqueue(pts, 0.0, 2)
            same(ctx.reach_matrix_wait(), RM.matrix(state, dist, (1, -2, 3), 0.1, pts, 0.0, 2, field_tiles(shape), ROUNDS), "field")
    ctx.close()


def test_terrain_matrix_jobs_change_nothing_else(tmp_path):
    def enable_a(a):
        a.terrain_enable(-2)
        a.reach_matrix_enable(8, field_tiles((64, 64, 32)), ROUNDS)

    def sites(t1):
        return [tuple(camera(t1 - 1) + d) for d in ((0.0, 0.0, 0.0), (1.0, 0.0, 2.0), (-1.0, 0.5, 3.0))]

    def enqueue(c, is_a, call, t1):
        if is_a:
            c.terrain_enqueue(1 + call % 3, 1)
            c.reach_matrix_enqueue_terrain(sites(t1), 0.0, 2)

    def check(a, outs, call, t1, what):
        state, origin = outs["state"][0], outs["field"][1]
        tr = a.terrain_wait()
        known_space.same(tr, TR.job(state, origin, 0.1, -2, 1 + call % 3, 1), what, TNAMES)
        same(a.reach_matrix_wait(), RMT.matrix(tr, 0.1, sites(t1), 0.0, 2, field_tiles((64, 64, 32)), ROUNDS), what)

    twin_drive(tmp_path, lambda c: None, enable_a, enqueue, lambda c: {}, check)


# ---- the ground chain on the synthetic road ----
def test_ground_chain_on_the_synthetic_road():
    """terrain(5, 1), frontiers, a terrain reach job with frontiers from the road 8 m ahead, the matrix over that start
    and the reached viewpoint cells' centres, then the tour: asserted on the model, then the device equals the model."""
    ctx, state, origin = road_scene.road_request()
    voxel, shape = road_scene.ROAD_VOXEL, road_scene.ROAD_SHAPE
    v = float(np.float32(voxel))
    ctx.terrain_enable(-2)
    ctx.frontier_enable(256, 1 << 18)
    ctx.reach_enable(255, 1 << 16, ROUNDS)
    ctx.reach_matrix_enable(256, field_tiles(shape), ROUNDS)
    ctx.tour_enable(256, 4)
    ctx.mcaps = (field_tiles(shape), ROUNDS, 256, -2, shape, voxel)
    tr = terrain(ctx, state, origin, 5, 1, "road")
    L, S = tr[1][:, 0, :], tr[2][:, 0, :]
    P = shape[0]
    ground = int(np.floor(1.65 / v)) - origin[1]
    xs = (np.arange(shape[0]) + origin[0] + 0.5) * v
    zs = (np.arange(shape[2]) + origin[2] + 0.5) * v
    road = np.argwhere((S == FREE) & (L == ground) & (np.abs(xs) <= 1.0)[None, :])
    z, x = road[np.argmin(np.abs(zs[road[:, 0]] - 8.0) + np.abs(xs[road[:, 1]]))]
    start = (xs[x], 1.6, zs[z])
    ctx.frontier_enqueue(1)
    fc, fv, _ = ctx.frontier_wait()
    ctx.reach_enqueue_terrain(start, 0.0, 2, None, True)
    rgot = ctx.reach_wait()
    rwant = RT.job(tr, shape, voxel, start, 0.0, 2, (), (fc, fv), 255, 1 << 16, ROUNDS)
    known_space.same(rgot, rwant, "road reach", ("header", "targets", "path list", "cost grid"))
    recs = rwant[1]
    hit = recs[recs["status"] == 0]
    assert len(hit) > 2
    pts = [start] + cell_centres(hit["viewpoint"], tr, voxel, 1.6)
    info, sites, M = RMT.matrix(tr, voxel, pts, 0.0, 2, field_tiles(shape), ROUNDS, 256)
    # the model: every site snaps to its own cell, row 0 is the reach job's costs, entries bound below by the chamfer
    assert (sites["status"] == 0).all() and (sites["approach"] == 0).all()
    assert sites["voxel"][0] == rwant[0]["start_voxel"] and (sites["voxel"][1:] == hit["viewpoint"]).all()
    assert (M[0, 1:].astype(np.int64) == hit["cost"].astype(np.int64) - hit["approach"]).all()
    c = sites["voxel"].astype(np.int64)
    dp, dq = np.abs((c % P)[:, None] - (c % P)[None, :]), np.abs((c // P)[:, None] - (c // P)[None, :])
    chamfer = 10 * np.maximum(dp, dq) + 4 * np.minimum(dp, dq)
    assert (M.astype(np.int64) >= chamfer).all() and (sites["converged"] == 1).all()
    tinfo, starts, order = TM.tour(M, 1, 4, 16, 7)
    reached = set(np.flatnonzero(M[0] != R.INF).tolist())
    assert set(order[:tinfo["n_included"]].tolist()) == reached and tinfo["n_infinite"] == 0
    # the device
    got = mjob(ctx, tr, pts, 0.0, 2, what="road matrix")
    ctx.tour_enqueue(got[2], 1, 4, 16, 7)
    known_space.same(ctx.tour_wait(), (tinfo, starts, order), "road tour", ("header", "starts", "order"))
    ctx.close()


# ---- the rejected frame and the error contract ----
def test_rejected_frame_comes_back_from_wait():
    def sites(first):
        return [tuple(camera(first - 1)), tuple(camera(first - 1) + (1.0, 0.0, 1.0))]

    def enqueue(b, first):
        b.terrain_enqueue(3, 1)
        b.reach_matrix_enqueue_terrain(sites(first), 0.0, 2)

    r = rejected_known(lambda b: (b.terrain_enable(-2), b.reach_matrix_enable(4, field_tiles((64, 64, 32)), ROUNDS)), enqueue)
    e = rejected(r.ctx.reach_matrix_wait)
    tr = rejected(r.ctx.terrain_wait).terrain
    known_space.same(tr, TR.job(r.state, r.field[1], r.voxel, -2, 3, 1), "rejected terrain", TNAMES)
    same(e.reach_matrix, RMT.matrix(tr, r.voxel, sites(r.first), 0.0, 2, field_tiles(r.shape), ROUNDS), "rejected")
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    pts = np.zeros((3, 3))
    enq = lambda c, p=pts.ctypes.data, n=1, radius=0.0, k=0: lib.dsm_reach_matrix_enqueue_terrain(c, p, n, radius, k)
    assert enq(None) == -1
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 12, 8)
    ctx.views_enable(1, 1.0)
    ctx.terrain_enable(3)
    assert enq(ctx.h) == -7                                  # before dsm_reach_matrix_enable
    ctx.reach_matrix_enable(2, 4, 64)                        # the field has 2 x 2 x 1 tiles
    assert enq(ctx.h) == -7                                  # no terrain job yet
    st = np.full((8, 12, 16), FREE, np.uint8)
    st[0] = OCCUPIED
    ctx.debug_field_load_state(st, (0, 0, 0))
    ctx.field_wait()
    assert enq(ctx.h) == -7                                  # a field request is no terrain job
    ctx.terrain_enqueue(2, 0)                                # in flight: a job may run behind it
    bad = np.array([[0.0, float("nan"), 0.0]])
    for kw in (dict(radius=float("nan")), dict(radius=-1.0), dict(radius=float("inf")), dict(k=-1), dict(k=5), dict(n=0), dict(n=3),
               dict(n=-1), dict(p=None), dict(p=bad.ctypes.data)):
        assert enq(ctx.h, **kw) == -1, kw
    assert enq(ctx.h, n=2) == 0                              # n_points = max_sites
    assert enq(ctx.h) == -7                                  # one matrix job in flight
    assert lib.dsm_reach_matrix_enqueue(ctx.h, pts.ctypes.data, 1, 0.0, 0) == -7
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == 0
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == -7
    ctx.terrain_wait()
    ctx.close()
    # the work bound: n_points x max_tiles x max_rounds <= 2^32 with max_tiles = 4096 (the field's 64 x 64 x 1 tiles)
    # and max_rounds = 65536
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 512, 512, 8)
    ctx.views_enable(1, 1.0)
    ctx.terrain_enable(3)
    ctx.reach_matrix_enable(17, 4096, 65536)
    st = np.full((8, 512, 512), FREE, np.uint8)
    st[0] = OCCUPIED
    ctx.debug_field_load_state(st, (0, 0, 0))
    ctx.field_wait()
    ctx.terrain_enqueue(2, 0)
    ctx.terrain_wait()
    big = np.zeros((17, 3))
    assert enq(ctx.h, p=big.ctypes.data, n=17) == -1
    assert enq(ctx.h, p=big.ctypes.data, n=16) == 0
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == 0
    ctx.close()


# ---- the node ----
def test_node_reach_matrix_terrain_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, terrain(), frontiers(), reach_terrain(with
    frontiers) from the field's middle and reach_matrix_terrain over that point and the reached viewpoint cells' centres
    equal the model over the grid the driver dumps; clouds, PLY and PCD files equal a twin without these jobs;
    reach_matrix_terrain() before terrain() on the frame and after load_state until the next fused frame returns
    DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    tiles = field_tiles((nx, ny, nz))
    r = run_driver("reach_matrix_terrain_main", str(tmp_path), cam, sc, node_args() + [32, tiles, 2048, RELOAD], tag="a", after=[pa])
    q = run_driver("reach_matrix_terrain_main", str(tmp_path), cam, sc, node_args() + [0, 0, 0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, k = r.i(), r.i()
        radius = float(r.take(np.float32, 1)[0])
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        pts = r.lst(np.float64).reshape(-1, 3)
        info = r.take(np.uint8, RM.MATRIX_INFO_DTYPE.itemsize).view(RM.MATRIX_INFO_DTYPE)[0].copy()
        sites = r.lst(RM.SITE_DTYPE)
        m = r.lst(np.uint32).reshape(len(sites), len(sites))
        before_terrain, after_load = r.i(), r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        tr = TR.job(state, origin, voxel, -2, 3, 1)
        same((info, sites, m), RMT.matrix(tr, voxel, pts, radius, k, tiles, 2048, 32), f"message {t}")
        found += int((m != R.INF).sum()) > len(sites)
        assert before_terrain == -7, f"message {t}"
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: reach_matrix_terrain() after load_state"
    assert found > 0
    twin_node_tail(r, q, pa, pb)
