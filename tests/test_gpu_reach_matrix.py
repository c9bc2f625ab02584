"""dsm_reach_matrix_enable / _enqueue / _wait: travel costs between many sites through the known free space of the
latest known field.

The device equals oracle/pyoracle_reach_matrix.matrix bit for bit in the header, the site records and the matrix: on every
known field of the windowed drive (sites: the field's centre, the viewpoints of a reach job with frontiers, random
points), with a resident twin of each request; on grids loaded through resident_map.load_known (hand cases, a density
sweep, a maze, the serpentine cut short, 128x128x72 converged against Dijkstra, n_points = max_sites).  Row i equals the
host-copy cost grid of a dsm_reach job started at site i, read at the sites, with that job's rounds, converged and
n_reached, converged and unconverged.  Both sides of the capacity cut, stream order against the next field request, a
drive with matrix jobs beside publish snapshots, checkpoints and reach jobs against a twin without them, the rejected
frame and every error code.  The node is checked through tests/cpp/reach_matrix_main.cpp."""
import ctypes
import filecmp

import numpy as np
import pytest
from scipy.sparse import csgraph

import pyoracle_reach as R
import pyoracle_reach_matrix as RM
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import SHAPES, STORE, T, camera, load_known, map_state, new_ctx, simple_lists, warp, windowed
from test_frontier_model import serpentine
from test_gpu_field_known import MAX_RANGE, Views
from test_gpu_reach import maze

pytestmark = pytest.mark.gpu

SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
UNKNOWN, OCCUPIED, FREE = R.UNKNOWN, R.OCCUPIED, R.FREE


def same(got, want, what):
    gi, gs, gm = got
    wi, ws, wm = want
    assert gi.tobytes() == np.array(wi).tobytes(), f"{what}: header {gi} want {wi}"
    assert gs.tobytes() == ws.tobytes(), f"{what}: sites\n{gs}\nwant\n{ws}"
    assert gm.tobytes() == wm.tobytes(), f"{what}: {(gm != wm).sum()} of {gm.size} matrix entries differ"


def loader(shape, voxel=0.2, max_sites=64, max_tiles=None, max_rounds=4096, reach=None):
    """A context whose field has grid `shape` (nx, ny, nz), with views and matrix jobs enabled (max_tiles: every tile),
    and reach jobs with `reach` = (max_targets, max_path, max_rounds) capacities."""
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(1, 1.0)
    tiles = int(np.prod([(n + 7) // 8 for n in shape]))
    ctx.reach_matrix_enable(max_sites, tiles if max_tiles is None else max_tiles, max_rounds)
    if reach:
        ctx.reach_enable(*reach)
    ctx.mcaps = (tiles if max_tiles is None else max_tiles, max_rounds)
    return ctx


def job(ctx, state, dist, origin, voxel, points, radius, k, what=""):
    max_tiles, max_rounds = ctx.mcaps
    ctx.reach_matrix_enqueue(points, radius, k)
    got = ctx.reach_matrix_wait()
    same(got, RM.matrix(state, dist, origin, voxel, points, radius, k, max_tiles, max_rounds), what)
    return got


def loaded(ctx, state, origin, voxel, points, radius, k, what=""):
    dist = load_known(ctx, state, origin, voxel, what)
    return job(ctx, state, dist, origin, voxel, points, radius, k, what)


def world(c, origin, voxel):
    return tuple((c[i] + origin[i] + 0.5) * float(np.float32(voxel)) for i in range(3))


def test_hand_cases():
    st = np.full((6, 12, 12), FREE, np.uint8)
    st[:, :, 6] = OCCUPIED
    st[:, 11, 6] = FREE
    st[3, 3, 9] = OCCUPIED
    o, v = (2, -3, 0), 0.5
    pts = [world(c, o, v) for c in [(1, 1, 1), (2, 1, 1), (9, 3, 3), (1, 1, 1), (20, 0, 0), (10, 2, 2), (-1, 5, 5), (11, 11, 5)]]
    ctx = loader((12, 12, 6), v, max_sites=8)
    for k in range(5):
        for radius in (0.0, 0.5, 1.0, 10.0):
            loaded(ctx, st, o, v, pts, radius, k, f"wall k={k} r={radius}")
    ctx.close()
    for shape in [(1, 1, 1), (7, 1, 1), (1, 9, 3), (9, 17, 8)]:   # axes of one voxel, tile edges
        ctx = loader(shape, 0.2, max_sites=16)
        rng = np.random.default_rng(sum(shape))
        for p in [(0.2, 0.1, 0.7), (0.0, 0.0, 1.0)]:
            st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
            pts = [world(rng.integers(-1, np.array(shape) + 1), (0, 0, 0), 0.2) for _ in range(16)]
            for k in (0, 2):
                loaded(ctx, st, (0, 0, 0), 0.2, pts, 0.0, k, f"{shape} {p} k={k}")
        ctx.close()


def test_density_sweep_and_a_full_site_table():
    shape, voxel, o = (64, 48, 24), 0.2, (-30, -20, -4)
    ctx = loader(shape, voxel, max_sites=24)
    rng = np.random.default_rng(21)
    for p in [(0.1, 0.1, 0.8), (0.2, 0.1, 0.7), (0.3, 0.1, 0.6), (0.05, 0.3, 0.65), (0.0, 0.5, 0.5)]:
        st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
        dist = load_known(ctx, st, o, voxel, f"density {p}")
        for radius, k, n in [(0.0, 0, 24), (0.2, 2, 9), (0.25, 4, 1)]:
            pts = [world(rng.integers(-2, np.array(shape) + 2), o, voxel) for _ in range(n)]
            job(ctx, st, dist, o, voxel, pts, radius, k, f"density {p} r={radius} k={k} n={n}")
    ctx.close()


def test_maze_and_the_serpentine_cut_short():
    st = maze(40, 3)
    nz, ny, nx = st.shape
    ctx = loader((nx, ny, nz), 0.1, max_sites=6)
    pts = [world(c, (0, 0, 0), 0.1) for c in [(1, 1, 0), (nx - 2, ny - 2, 0), (1, ny - 2, 1), (nx - 2, 1, 0), (41, 41, 1), (3, 1, 1)]]
    got = loaded(ctx, st, (0, 0, 0), 0.1, pts, 0.0, 0, "maze")
    assert (got[1]["converged"] == 1).all() and (got[2] == got[2].T).all()
    ctx.close()
    sp = serpentine(48, 40, 8)
    for rounds in (1, 7, 40):
        ctx = loader((48, 40, 8), 0.2, max_sites=8, max_rounds=rounds)
        pts = [world(c, (3, -2, 1), 0.2) for c in [(0, 0, 0), (47, 39, 7), (47, 0, 0), (0, 2, 0), (20, 38, 0), (5, 0, 2), (0, 0, 6), (0, 0, 0)]]
        got = loaded(ctx, sp, (3, -2, 1), 0.2, pts, 0.0, 1, f"serpentine, {rounds} rounds")
        assert (got[1]["converged"] == 0).any()
        ctx.close()


def test_a_large_grid_converged_against_dijkstra():
    shape, voxel, o = (128, 128, 72), 0.1, (-64, -64, -10)
    rng = np.random.default_rng(8)
    st = rng.choice(3, size=shape[::-1], p=(0.03, 0.12, 0.85)).astype(np.uint8)
    ctx = loader(shape, voxel, max_sites=32)
    dist = load_known(ctx, st, o, voxel, "128x128x72")
    trav = R.traversable(st, dist, 0.1)
    u = rng.choice(np.flatnonzero(trav.reshape(-1)), size=32, replace=False)
    nz, ny, nx = st.shape
    pts = [world((x % nx, x // nx % ny, x // (nx * ny)), o, voxel) for x in u.tolist()]
    ctx.reach_matrix_enqueue(pts, 0.1, 1)
    info, sites, M = ctx.reach_matrix_wait()
    assert info["status"] == 0 and (sites["status"] == 0).all() and (sites["converged"] == 1).all()
    assert sites["voxel"].tolist() == u.tolist() and (sites["approach"] == 0).all()
    d = csgraph.dijkstra(R.graph(trav), directed=False, indices=u)[:, u]
    assert M.tobytes() == np.where(np.isfinite(d), d, R.INF).astype(np.uint32).tobytes()
    assert info["n_active_tiles"] == RM.active_tiles(trav).sum() and info["n_traversable"] == trav.sum()
    ctx.close()


@pytest.mark.parametrize("rounds", [7, 4096])
def test_rows_equal_single_source_reach_jobs(rounds):
    """Two device paths: row i of a matrix job equals the host-copy cost grid of a dsm_reach job started at site i on the
    same field, read at the sites, and that job's rounds, converged and n_reached."""
    cases = [((48, 40, 8), serpentine(48, 40, 8)), ((40, 33, 17), None)]
    rng = np.random.default_rng(rounds)
    for shape, st in cases:
        if st is None:
            st = rng.choice(3, size=shape[::-1], p=(0.15, 0.1, 0.75)).astype(np.uint8)
        ctx = loader(shape, 0.2, max_sites=10, max_rounds=rounds, reach=(4, 1 << 12, rounds))
        load_known(ctx, st, (0, 0, 0), 0.2)
        pts = [world(rng.integers(0, shape), (0, 0, 0), 0.2) for _ in range(9)] + [(-5.0, 0.0, 0.0)]
        for radius, k in [(0.0, 1), (0.2, 3)]:
            ctx.reach_matrix_enqueue(pts, radius, k)
            info, sites, M = ctx.reach_matrix_wait()
            u = sites["voxel"]
            for i, p in enumerate(pts):
                ctx.reach_enqueue(p, radius, k, None, False, True)
                ri, _, _, cost = ctx.reach_wait()
                what = f"{shape} rounds={rounds} r={radius} k={k} site {i}"
                assert (ri["start_voxel"], ri["start_status"], ri["start_approach"]) == tuple(sites[i][["voxel", "status", "approach"]].tolist()), what
                assert (ri["rounds"], ri["converged"], ri["n_reached"]) == tuple(sites[i][["rounds", "converged", "n_reached"]].tolist()), what
                want = np.where(u >= 0, cost.reshape(-1)[np.maximum(u, 0)], R.INF).astype(np.uint32) if u[i] >= 0 else np.full(len(u), R.INF, np.uint32)
                assert M[i].tobytes() == want.tobytes(), what
            assert rounds != 7 or shape != (48, 40, 8) or (sites["converged"][sites["status"] == 0] == 0).any()
        ctx.close()


def test_both_sides_of_the_capacity_cut():
    shape = (30, 20, 12)
    rng = np.random.default_rng(5)
    st = rng.choice(3, size=shape[::-1], p=(0.2, 0.2, 0.6)).astype(np.uint8)
    trav = R.traversable(st, np.full(st.shape, np.inf, np.float32), 0.0)
    n_active = int(RM.active_tiles(trav).sum())
    pts = [world(rng.integers(0, shape), (0, 0, 0), 0.2) for _ in range(7)]
    for max_tiles in (n_active, n_active - 1, 1):
        ctx = loader(shape, 0.2, max_sites=7, max_tiles=max_tiles)
        got = loaded(ctx, st, (0, 0, 0), 0.2, pts, 0.0, 1, f"max_tiles {max_tiles} of {n_active}")
        assert got[0]["status"] == int(max_tiles < n_active)
        # a larger radius leaves fewer active tiles: the same context passes
        st2 = st.copy()
        st2[:, :, 8:] = OCCUPIED
        st2[:, 8:, :] = OCCUPIED
        st2[8:, :, :] = OCCUPIED
        got = loaded(ctx, st2, (0, 0, 0), 0.2, pts, 0.0, 1, f"one tile, max_tiles {max_tiles}")
        assert got[0]["status"] == 0 and got[0]["n_active_tiles"] <= 1
        ctx.close()


def test_stream_order():
    """A job reads the field it was enqueued behind, not the next field request."""
    shape, voxel = (40, 30, 20), 0.2
    ctx = loader(shape, voxel, max_sites=12)
    rng = np.random.default_rng(9)
    a = rng.choice(3, size=shape[::-1], p=(0.1, 0.1, 0.8)).astype(np.uint8)
    b = rng.choice(3, size=shape[::-1], p=(0.3, 0.1, 0.6)).astype(np.uint8)
    pts = rng.uniform(0, 4, size=(12, 3))
    ctx.debug_field_load_state(a, (0, 0, 0))
    ctx.reach_matrix_enqueue(pts, 0.0, 1)                  # before the field is waited for
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_matrix_enqueue(pts, 0.0, 1)              # one job in flight
    assert e.value.code == -7
    da = ctx.field_wait()[0]
    got = ctx.reach_matrix_wait()
    want = RM.matrix(a, da, (0, 0, 0), voxel, pts, 0.0, 1, *ctx.mcaps)
    same(got, want, "first")
    ctx.reach_matrix_enqueue(pts, 0.0, 1)
    ctx.debug_field_load_state(b, (5, 5, 5))               # the next request, while the job is in flight
    got = ctx.reach_matrix_wait()
    db = ctx.field_wait()[0]
    same(got, want, "the old field")
    ctx.reach_matrix_enqueue(pts, 0.0, 1)
    same(ctx.reach_matrix_wait(), RM.matrix(b, db, (5, 5, 5), voxel, pts, 0.0, 1, *ctx.mcaps), "the new field")
    ctx.field_enqueue((0, 0, 0), 1)                        # a plain request
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_matrix_enqueue(pts, 0.0, 1)
    assert e.value.code == -7
    ctx.field_wait()
    ctx.close()


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_fields_of_the_drive(chunk, shape):
    """The windowed drive with loop-closure warps between calls; after every call a known field, its frontiers, a reach
    job from the camera to the clusters, and a matrix job over the field's centre, the reached viewpoints and random
    points, against the model on the field's own grids; the same job on a resident twin of the request equals it."""
    lists = simple_lists()
    voxels = (0.125, 0.1, 0.3)
    ctxs, views = {}, {}
    tiles = int(np.prod([(n + 7) // 8 for n in shape]))
    for v in voxels:
        ctxs[v] = new_ctx(store=STORE)
        ctxs[v].field_enable(v, *shape)
        views[v] = Views(ctxs[v], 6)
        ctxs[v].frontier_enable(64, 1 << 16)
        ctxs[v].reach_enable(16, 1 << 12, 2048)
        ctxs[v].reach_matrix_enable(16, tiles, 2048)
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
        dist, origin, _ = ctx.field_wait()
        state, _ = ctx.field_state()
        ctx.frontier_enqueue(1 + call % 3)
        ctx.frontier_wait()
        ctx.reach_enqueue(cam, 0.0, 1, None, True)
        _, targets, _, _ = ctx.reach_wait()
        nz, ny, nx = state.shape
        vp = targets["viewpoint"][targets["status"] == 0][:8].astype(np.int64)
        pts = [world((nx // 2, ny // 2, nz // 2), origin, v), tuple(cam)]
        pts += [world((x % nx, x // nx % ny, x // (nx * ny)), origin, v) for x in vp.tolist()]
        pts += [tuple(cam + rng.uniform(-2, 2, 3)) for _ in range(16 - len(pts))]
        k, radius = call % 5, (0.0, v, 2 * v)[call % 3]
        ctx.mcaps = (tiles, 2048)
        got = job(ctx, state, dist, origin, v, pts, radius, k, f"frames {t0}-{t1 - 1}, voxel {v}")
        seen += int((got[2][0] != R.INF).sum()) > 1
        ctx.field_enqueue_known(cam, 5, slots, poses, host_copy=False)   # a resident twin of the same request
        ctx.field_wait()
        ctx.reach_matrix_enqueue(pts, radius, k)
        twin = ctx.reach_matrix_wait()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(twin, got)), "resident twin"
    assert seen > 0 or shape == (1, 1, 1)
    for c in ctxs.values():
        c.close()


def test_matrix_jobs_change_nothing_else(tmp_path):
    """A drive with frontier, reach and matrix jobs beside a publish snapshot and an asynchronous checkpoint leaves the
    map, both published clouds, the fields, the state grids, the frontiers, the reach results and the checkpoint files
    byte-identical to a twin without matrix jobs."""
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
        c.reach_enable(64, 1 << 14, 1024)
    a.reach_matrix_enable(8, 8 * 8 * 4, 1024)
    stored = set()
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        for c, d in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            d["v"].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        outs = []
        pts = [camera(t) for t in range(t1)][-8:]
        for c, d in ((a, va), (b, vb)):
            slots, poses = d["v"].request()
            c.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
            c.frontier_enqueue(1)
            if c is a:
                a.reach_matrix_enqueue(pts, 0.1, 2)
            c.reach_enqueue(camera(t1 - 1), 0.1, 2, [camera(0)], True, True)
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
        got = a.reach_matrix_wait()
        fa, fb = outs[0][0], outs[1][0]
        what = f"after frames {t0}-{t1 - 1}"
        same(got, RM.matrix(outs[0][1][0], fa[0], fa[1], voxel, pts, 0.1, 2, 8 * 8 * 4, 1024), what)
        assert fa[0].tobytes() == fb[0].tobytes() and outs[0][1][0].tobytes() == outs[1][1][0].tobytes(), f"{what}: field"
        assert all(x.tobytes() == y.tobytes() for x, y in zip(outs[0][3], outs[1][3])), f"{what}: frontiers"
        assert all(x.tobytes() == y.tobytes() for x, y in zip(outs[0][4], outs[1][4])), f"{what}: reach"
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
    b.reach_matrix_enable(4, 8 * 8 * 4, 512)
    for call, t0 in enumerate(range(0, first + 2)):
        windowed(b, t0, t0 + 1, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 1)
    slots, poses = views.request()
    b.field_enqueue_known(camera(first - 1), 1, slots, poses)
    pts = [camera(0), camera(first - 1), camera(first - 1) + 1.0]
    b.reach_matrix_enqueue(pts, 0.0, 1)
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6
    dist, origin, _ = e.value.field
    state, _ = b.field_state()
    with pytest.raises(capi.DsmError) as e:
        b.reach_matrix_wait()
    assert e.value.code == -6
    same(e.value.reach_matrix, RM.matrix(state, dist, origin, voxel, pts, 0.0, 1, 8 * 8 * 4, 512), "rejected")
    assert (e.value.reach_matrix[1]["n_reached"] > 0).any()
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    b.close()


def test_error_contract():
    lib = capi.load_library()
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    st = np.full((4, 5, 6), FREE, np.uint8)
    p1 = np.zeros((1, 3))
    p3 = np.full((3, 3), 0.1)
    assert lib.dsm_reach_matrix_enable(ctx.h, 1, 1, 1) == -7                 # before dsm_field_enable
    ctx.field_enable(0.2, 6, 5, 4)
    assert lib.dsm_reach_matrix_enable(ctx.h, 1, 1, 1) == -7                 # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert lib.dsm_reach_matrix_enqueue(ctx.h, p1.ctypes.data, 1, 0.0, 0) == -7   # before dsm_reach_matrix_enable
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == -7
    for ms, mt, mr in [(0, 1, 1), (1025, 1, 1), (-1, 1, 1), (1, 0, 1), (1, 2, 1), (1, 1, 0), (1, 1, R.MAX_ROUNDS + 1)]:
        assert lib.dsm_reach_matrix_enable(ctx.h, ms, mt, mr) == -1, (ms, mt, mr)   # one tile in a 6x5x4 grid
    assert lib.dsm_reach_matrix_enable(None, 1, 1, 1) == -1
    big = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    big.pool_upload(np.zeros(0, SURFEL_DTYPE))
    big.field_enable(0.2, 8 * 65, 8 * 64, 8)                                 # 4160 tiles
    big.views_enable(1, 1.0)
    assert lib.dsm_reach_matrix_enable(big.h, 1024, 4097, 1) == -1          # 4 KB x 1024 x 4097 > 2^34 B
    assert lib.dsm_reach_matrix_enable(big.h, 1, 4161, 1) == -1             # more slots than tiles
    big.close()
    ctx.reach_matrix_enable(3, 1, 2)
    assert lib.dsm_reach_matrix_enable(ctx.h, 1, 1, 1) == -7                 # once
    assert lib.dsm_reach_matrix_enqueue(ctx.h, p1.ctypes.data, 1, 0.0, 0) == -7   # no field request yet
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == -7          # nothing enqueued
    ctx.field_enqueue((0, 0, 0), 1)                                          # a plain request
    ctx.field_wait()
    assert lib.dsm_reach_matrix_enqueue(ctx.h, p1.ctypes.data, 1, 0.0, 0) == -7
    load_known(ctx, st, (0, 0, 0), 0.2)
    nan, inf = float("nan"), float("inf")
    for pts, n, radius, k in [(np.array([[nan, 0, 0]]), 1, 0.0, 0), (np.array([[0, inf, 0]]), 1, 0.0, 0), (p1, 1, -0.1, 0),
                              (p1, 1, nan, 0), (p1, 1, inf, 0), (p1, 1, 0.0, -1), (p1, 1, 0.0, 5), (p1, 0, 0.0, 0),
                              (p3, 4, 0.0, 0), (p3, -1, 0.0, 0), (None, 1, 0.0, 0)]:
        assert lib.dsm_reach_matrix_enqueue(ctx.h, None if pts is None else pts.ctypes.data, n, radius, k) == -1, (pts, n, radius, k)
    assert lib.dsm_reach_matrix_enqueue(None, p1.ctypes.data, 1, 0.0, 0) == -1
    assert lib.dsm_reach_matrix_enqueue(ctx.h, p3.ctypes.data, 3, 0.0, 4) == 0
    assert lib.dsm_reach_matrix_enqueue(ctx.h, p3.ctypes.data, 3, 0.0, 4) == -7   # one job in flight
    info = np.zeros(1, capi.REACH_MATRIX_INFO_DTYPE)
    assert lib.dsm_reach_matrix_wait(ctx.h, info.ctypes.data, None, None) == 0
    assert info[0]["n_traversable"] == st.size and info[0]["n_sites"] == 3 and info[0]["n_active_tiles"] == 1
    assert lib.dsm_reach_matrix_wait(ctx.h, None, None, None) == -7
    ctx.close()
    # the work bound: n_points x max_tiles x max_rounds above 2^32 tile relaxations
    w = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    w.pool_upload(np.zeros(0, SURFEL_DTYPE))
    w.field_enable(0.2, 8 * 64, 8 * 64, 8)                                   # 4096 tiles
    w.views_enable(1, 1.0)
    w.reach_matrix_enable(17, 4096, 65536)
    w.debug_field_load_state(np.full((8, 512, 512), FREE, np.uint8), (0, 0, 0))
    w.field_wait()
    pts = np.full((17, 3), 0.1)
    assert lib.dsm_reach_matrix_enqueue(w.h, pts.ctypes.data, 17, 0.0, 0) == -1   # 17 x 2^12 x 2^16 > 2^32
    assert lib.dsm_reach_matrix_enqueue(w.h, pts.ctypes.data, 16, 0.0, 0) == 0    # 2^32 exactly
    w.reach_matrix_wait()
    w.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)
MAX_VIEWS = 5
RELOAD = 12   # the node saves and loads its state after this depth message


def test_node_reach_matrix_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers(), reach(with_frontiers) from the
    field's centre and reach_matrix over that point and the reached viewpoints: the snaps equal the model's and the
    converged matrix equals Dijkstra's over the grids the driver dumps; clouds, PLY and PCD files equal a twin without matrix jobs; reach_matrix after load_state until the
    next fused frame returns DSM_E_STATE."""
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    node = [2, 0, 1 << 20, 1 << 21, *FIELD, MAX_VIEWS, MAX_RANGE]
    tiles = 12 * 12 * 4
    r = run_driver("reach_matrix_main", str(tmp_path), cam, sc, node + [32, tiles, 2048, RELOAD], tag="a", after=[pa])
    q = run_driver("reach_matrix_main", str(tmp_path), cam, sc, node + [0, 0, 0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, k = r.i(), r.i()
        radius = float(r.take(np.float32, 1)[0])
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        pts = r.lst(np.float64).reshape(-1, 3)
        info = r.take(np.uint8, RM.MATRIX_INFO_DTYPE.itemsize).view(RM.MATRIX_INFO_DTYPE)[0].copy()
        sites = r.lst(RM.SITE_DTYPE)
        m = r.lst(np.uint32)
        after_load = r.i()
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == 0 and rr == 0 and rq == 0, f"message {t}: {rc} {rr} {rq}"
        # every job converges well within 2048 rounds here, so the model's rows are Dijkstra's (emulating each row on the
        # host would take minutes per drive)
        what = f"message {t}"
        trav = R.traversable(state, dist, radius)
        snaps = [R.snap(trav, R.voxel_of(p, origin, voxel, (nx, ny, nz)), k) for p in pts]
        assert [tuple(x) for x in sites[["voxel", "status", "approach"]].tolist()] == snaps, what
        assert (sites["converged"] == 1).all() and info["status"] == 0 and info["n_sites"] == len(pts), what
        assert info["n_traversable"] == trav.sum() and info["n_active_tiles"] == RM.active_tiles(trav).sum(), what
        u = sites["voxel"]
        d = csgraph.dijkstra(R.graph(trav), directed=False, indices=np.maximum(u, 0))[:, np.maximum(u, 0)]
        want = np.where(np.isfinite(d) & (u[:, None] >= 0) & (u[None, :] >= 0), d, R.INF).astype(np.uint32)
        assert m.tobytes() == want.tobytes(), f"{what}: {(m.reshape(want.shape) != want).sum()} entries differ"
        found += int((m != R.INF).sum()) > len(sites)
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: reach_matrix() after load_state"
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
    assert found > 0
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
