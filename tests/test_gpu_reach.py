"""dsm_reach_enable / _enqueue / _wait: travel cost through the known free space of the latest known field.

The device equals oracle/pyoracle_reach bit for bit in the whole header (rounds and converged included), the target
records, the path list and the cost grid: on every known field of the windowed drive, with frontier targets (the model
runs on the device's own field_wait / field_state, which tests/test_gpu_field_known.py pins to the known-space oracle);
on grids loaded through dsm_debug_field_load_state (hand cases, random grids over a sweep of densities, a maze, a
serpentine cut short by max_rounds against the round emulator, a grid of over a million voxels against Dijkstra; each
load's distances, counts and states are held to the known-space oracle first, through resident_map.load_known); a
resident job equals its host-copy twin; the stream order against the next field request and the next frontier job; a
drive with reach jobs beside publish snapshots and asynchronous checkpoints leaves everything as a twin without them;
the rejected-frame and error contracts.  The node is checked through tests/cpp/reach_main.cpp."""
import ctypes
from functools import partial

import numpy as np
import pytest

import known_space
import pyoracle_frontier
import pyoracle_reach as R
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, NODE_FIELD, assert_error_stays, known_drive, node_args,
                         rejected, rejected_known, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import maze, serpentine
from resident_map import SHAPES, camera, load_known

pytestmark = pytest.mark.gpu

FRONTIER_CAPS = (256, 1 << 18)
same = partial(known_space.same, names=("header", "targets", "path list", "cost grid"))


def loader(shape, voxel=0.2, caps=(64, 1 << 16), max_rounds=4096, frontier_caps=FRONTIER_CAPS):
    """A context whose field has grid `shape` (nx, ny, nz), with views, frontiers and reach jobs enabled."""
    ctx = small_ctx(shape, voxel)
    ctx.frontier_enable(*frontier_caps)
    ctx.reach_enable(*caps, max_rounds)
    ctx.caps = (caps, max_rounds, frontier_caps)
    return ctx


def job(ctx, dist, state, origin, voxel, start, radius, k, goals=(), with_frontiers=False, m=1, host_copy=True, exact=False):
    """The device's job on the latest (waited) known field against the model on its dist and state grids."""
    (mt, mp), mr, fcaps = ctx.caps
    fr = None
    if with_frontiers:
        ctx.frontier_enqueue(m)
        fc, fv, _ = ctx.frontier_wait()
        fr = (fc, fv)
    ctx.reach_enqueue(start, radius, k, goals, with_frontiers, host_copy)
    got = ctx.reach_wait()
    want = R.reach(state, dist, origin, voxel, start, radius, k, goals, fr, mt, mp, mr, exact)
    return got, want


def loaded(ctx, state, origin, voxel, start, radius, k, goals=(), with_frontiers=False, m=1, exact=False, what=""):
    dist = load_known(ctx, state, origin, voxel, what)
    got, want = job(ctx, dist, state, origin, voxel, start, radius, k, goals, with_frontiers, m, exact=exact)
    same(got, want, what, rounds=not exact)
    return got


def world(c, origin, voxel):
    return tuple((c[i] + origin[i] + 0.5) * float(np.float32(voxel)) for i in range(3))


def test_hand_cases():
    voxel, o = 0.5, (-3, 2, 1)
    st = np.full((4, 4, 4), FREE, np.uint8)
    st[:, :, 2] = OCCUPIED
    ctx = loader((4, 4, 4), voxel)
    goals = [world(c, o, voxel) for c in [(3, 3, 3), (-1, 0, 0), (2, 3, 3), (0, 0, 0), (1, 3, 0)]]
    for k in range(5):
        for radius in (0.0, 0.5, np.float32(0.5) + np.float32(1e-7), 1.0, 10.0):   # 0.5 a stored distance: v
            for start in [world((0, 0, 0), o, voxel), world((3, 3, 3), o, voxel), world((2, 1, 1), o, voxel), (-50.0, 0.0, 0.0)]:
                loaded(ctx, st, o, voxel, start, radius, k, goals, what=f"wall k={k} r={radius} start={start}")
    ctx.close()
    # ties: the snap, the viewpoint and the predecessor (a 3x3x3 box with an occupied centre), and a free 3x3x1 sheet
    for shape, st, starts in [((3, 3, 3), np.full((3, 3, 3), FREE, np.uint8), [(1, 1, 1), (0, 0, 0), (2, 2, 2)]),
                              ((3, 3, 1), np.full((1, 3, 3), FREE, np.uint8), [(0, 0, 0), (1, 1, 0)])]:
        if shape == (3, 3, 3):
            st[1, 1, 1] = OCCUPIED
        ctx = loader(shape, voxel)
        goals = [world(c, (0, 0, 0), voxel) for c in np.ndindex(*shape)]
        for s in starts:
            for k in (0, 1, 2):
                loaded(ctx, st, (0, 0, 0), voxel, world(s, (0, 0, 0), voxel), 0.0, k, goals, with_frontiers=True, what=f"{shape} {s} k={k}")
        ctx.close()
    # two one-voxel clusters, too close to the unknown ends to be traversable, reach the start (2) at the same cost
    st = np.full((1, 1, 5), FREE, np.uint8)
    st[0, 0, [0, 4]] = UNKNOWN
    ctx = loader((5, 1, 1), voxel)
    got = loaded(ctx, st, (0, 0, 0), voxel, world((2, 0, 0), (0, 0, 0), voxel), 1.0, 1, with_frontiers=True, what="member tie")
    assert got[1]["target"].tolist() == [1, 3] and got[1]["viewpoint"].tolist() == [2, 2] and got[1]["cost"].tolist() == [10, 10]
    ctx.close()
    for shape in [(1, 1, 1), (7, 1, 1), (1, 9, 3), (9, 17, 8)]:   # axes of one voxel, tile edges
        ctx = loader(shape, 0.2)
        rng = np.random.default_rng(sum(shape))
        for p in [(0.2, 0.1, 0.7), (0.0, 0.0, 1.0)]:
            st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
            goals = [world(rng.integers(-1, np.array(shape) + 1), (0, 0, 0), 0.2) for _ in range(6)]
            for k in (0, 2):
                loaded(ctx, st, (0, 0, 0), 0.2, world((0, 0, 0), (0, 0, 0), 0.2), 0.0, k, goals, with_frontiers=True, what=f"{shape} {p}")
        ctx.close()


def test_random_grids_over_a_density_sweep():
    shape, voxel, o = (64, 48, 24), 0.2, (-30, -20, -4)
    ctx = loader(shape, voxel, caps=(96, 1 << 14))
    rng = np.random.default_rng(21)
    for p in [(0.1, 0.1, 0.8), (0.2, 0.1, 0.7), (0.3, 0.1, 0.6), (0.05, 0.3, 0.65), (0.0, 0.5, 0.5)]:
        st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
        for radius, k in [(0.0, 0), (0.2, 2), (0.25, 4)]:
            start = world(rng.integers(0, shape), o, voxel)
            goals = [world(rng.integers(-2, np.array(shape) + 2), o, voxel) for _ in range(20)]
            loaded(ctx, st, o, voxel, start, radius, k, goals, with_frontiers=True, m=1 + k, what=f"density {p} r={radius} k={k}")
    ctx.close()


def test_maze():
    st = maze(40, 3)
    nz, ny, nx = st.shape
    ctx = loader((nx, ny, nz), 0.1, caps=(8, 1 << 16))
    corners = [world(c, (0, 0, 0), 0.1) for c in [(nx - 2, ny - 2, 0), (1, ny - 2, 1), (nx - 2, 1, 0), (41, 41, 1)]]
    loaded(ctx, st, (0, 0, 0), 0.1, world((1, 1, 0), (0, 0, 0), 0.1), 0.0, 0, corners, what="maze")
    ctx.close()


def test_serpentine_cut_short_and_a_million_voxels_converged():
    st = serpentine(48, 40, 8)
    ctx = loader((48, 40, 8), 0.2, caps=(16, 1 << 16), max_rounds=7)
    goals = [world(c, (0, 0, 0), 0.2) for c in [(47, 0, 0), (0, 2, 0), (20, 38, 0), (5, 0, 2), (0, 0, 6)]]
    got = loaded(ctx, st, (0, 0, 0), 0.2, world((0, 0, 0), (0, 0, 0), 0.2), 0.0, 1, goals, with_frontiers=True, what="serpentine, 7 rounds")
    assert got[0]["converged"] == 0 and got[0]["rounds"] == 7
    ctx.close()
    for rounds in (1, 40, 300):
        ctx = loader((48, 40, 8), 0.2, caps=(16, 1 << 16), max_rounds=rounds)
        loaded(ctx, st, (3, -2, 1), 0.2, world((47, 39, 7), (3, -2, 1), 0.2), 0.0, 2, goals, what=f"serpentine, {rounds} rounds")
        ctx.close()
    shape, voxel, o = (128, 128, 72), 0.1, (-64, -64, -10)
    rng = np.random.default_rng(8)
    st = rng.choice(3, size=shape[::-1], p=(0.03, 0.12, 0.85)).astype(np.uint8)
    assert st.size >= 1 << 20
    ctx = loader(shape, voxel, caps=(64, 1 << 16), max_rounds=4096)
    goals = [world(rng.integers(0, shape), o, voxel) for _ in range(40)]
    got = loaded(ctx, st, o, voxel, world((64, 64, 36), o, voxel), 0.1, 1, goals, exact=True, what="a million voxels")
    assert got[0]["n_reached"] > st.size // 2
    ctx.close()


def test_a_start_walled_off_in_its_tile():
    """The start is the only traversable voxel of its 8x8x8 tile, on a tile face, edge or corner, so it reaches the grid
    only across the tile's faces: the device equals the emulator, and its converged costs equal Dijkstra's."""
    cases = []
    st = np.full((1, 1, 20), FREE, np.uint8)
    st[0, 0, :7] = OCCUPIED
    cases.append((st, (7, 0, 0), [(19, 0, 0), (0, 0, 0)]))
    st = np.full((16, 16, 16), FREE, np.uint8)
    st[:8, :8, :8] = OCCUPIED
    st[7, 7, 7] = FREE
    cases.append((st, (7, 7, 7), [(15, 15, 15), (8, 0, 0)]))
    rng = np.random.default_rng(12)
    for p in [(8, 8, 8), (7, 3, 20), (16, 15, 4), (23, 8, 15)]:    # (x, y, z): corners, edges and faces of tiles
        st = rng.choice([OCCUPIED, FREE], size=(24, 24, 24), p=(0.25, 0.75)).astype(np.uint8)
        x, y, z = p
        st[z // 8 * 8:z // 8 * 8 + 8, y // 8 * 8:y // 8 * 8 + 8, x // 8 * 8:x // 8 * 8 + 8] = OCCUPIED
        st[z, y, x] = FREE
        cases.append((st, p, [tuple(int(c) for c in rng.integers(0, 24, size=3)) for _ in range(8)]))
    for st, p, goals in cases:
        nz, ny, nx = st.shape
        ctx = loader((nx, ny, nz), 0.5)
        got = loaded(ctx, st, (0, 0, 0), 0.5, world(p, (0, 0, 0), 0.5), 0.0, 0, [world(g, (0, 0, 0), 0.5) for g in goals],
                     what=f"walled off at {p}")
        info, _, _, cost = got
        trav = R.traversable(st, np.full(st.shape, np.inf, np.float32), 0.0)
        assert info["converged"] == 1 and info["rounds"] >= 2 and info["n_reached"] > 1, f"{p}: {info}"
        assert cost.tobytes() == R.dijkstra(trav, int(info["start_voxel"])).tobytes(), f"{p}: costs differ from Dijkstra"
        ctx.close()


def test_resident_job_equals_its_host_copy_twin_and_repeats():
    shape = (40, 33, 17)
    ctx = loader(shape, 0.2)
    rng = np.random.default_rng(4)
    st = rng.choice(3, size=shape[::-1], p=(0.15, 0.1, 0.75)).astype(np.uint8)
    load_known(ctx, st, (0, 0, 0), 0.2)
    goals = rng.uniform(0, 6, size=(30, 3))
    outs = []
    for host_copy in (False, True, False):
        ctx.frontier_enqueue(2)
        ctx.frontier_wait()
        ctx.reach_enqueue((3.1, 3.3, 1.7), 0.2, 2, goals, True, host_copy)
        outs.append(ctx.reach_wait())
    assert outs[0][3] is None and outs[1][3] is not None
    for a in (outs[0], outs[2]):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a[:3], outs[1][:3])), "resident and host-copy jobs"
    ctx.close()


def test_stream_order():
    """A job reads the field and the frontier result it was enqueued behind, not the next field request or frontier
    job; with_frontiers needs a frontier job on the latest field request."""
    shape, voxel = (40, 30, 20), 0.2
    ctx = loader(shape, voxel)
    rng = np.random.default_rng(9)
    a = rng.choice(3, size=shape[::-1], p=(0.1, 0.1, 0.8)).astype(np.uint8)
    b = rng.choice(3, size=shape[::-1], p=(0.3, 0.1, 0.6)).astype(np.uint8)
    start, goals = (2.0, 2.0, 1.0), rng.uniform(0, 4, size=(10, 3))
    ctx.debug_field_load_state(a, (0, 0, 0))
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_enqueue(start, 0.0, 1, goals, True)      # no frontier job on this field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    ctx.reach_enqueue(start, 0.0, 1, goals, True)           # before the field is waited for
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_enqueue(start, 0.0, 1, goals)              # one job in flight
    assert e.value.code == -7
    da = ctx.field_wait()[0]
    fa = ctx.frontier_wait()
    got = ctx.reach_wait()
    want = R.reach(a, da, (0, 0, 0), voxel, start, 0.0, 1, goals, fa[:2], 64, 1 << 16, 4096)
    same(got, want, "first")
    ctx.frontier_enqueue(1)
    ctx.reach_enqueue(start, 0.0, 1, goals, True)
    ctx.debug_field_load_state(b, (5, 5, 5))                 # the next request, while the job is in flight
    got = ctx.reach_wait()
    db = ctx.field_wait()[0]
    fa2 = ctx.frontier_wait()
    same(got, want, "the old field")
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_enqueue(start, 0.0, 1, goals, True)        # the frontier job read the old field
    assert e.value.code == -7
    ctx.frontier_enqueue(1)
    ctx.reach_enqueue(start, 0.0, 1, goals, True)
    fb = ctx.frontier_wait()
    ctx.frontier_enqueue(3)                                  # the next frontier job, while the reach job is in flight
    got = ctx.reach_wait()
    ctx.frontier_wait()
    same(got, R.reach(b, db, (5, 5, 5), voxel, start, 0.0, 1, goals, fb[:2], 64, 1 << 16, 4096), "the old frontiers")
    ctx.field_enqueue((0, 0, 0), 1)                          # a plain request
    with pytest.raises(capi.DsmError) as e:
        ctx.reach_enqueue(start, 0.0, 1, goals)
    assert e.value.code == -7
    ctx.field_wait()
    ctx.close()


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_fields_of_the_drive(chunk, shape):
    """The windowed drive with loop-closure warps between calls; after every call a known field, its frontiers and a
    reach job from the camera to the clusters and a few goals, against the model on the field's own grids."""
    def enable(c):
        c.frontier_enable(64, 1 << 16)
        c.reach_enable(96, 1 << 16, 2048)

    seen = 0
    for call, t0, t1, ctx, v, cam, _, _, (dist, origin, _), state in known_drive(shape, chunk, (0.125, 0.1, 0.3), enable):
        goals = [cam + d for d in ([1.0, 0, 0], [0, 1.0, 0.5], [-2.0, 0.3, 1.0], [0, 0, 0])]
        k, radius = call % 5, (0.0, v, 2 * v)[call % 3]
        ctx.caps = ((96, 1 << 16), 2048, (64, 1 << 16))
        got, want = job(ctx, dist, state, origin, v, cam, radius, k, goals, True, 1 + call % 3)
        same(got, want, f"frames {t0}-{t1 - 1}, voxel {v}")
        seen += int((got[1]["status"] == 0).sum()) > 1
    assert seen > 0 or shape == (1, 1, 1)


def test_reach_jobs_change_nothing_else(tmp_path):
    """A drive with frontier and reach jobs beside a publish snapshot and an asynchronous checkpoint leaves the map,
    both published clouds, the fields, the state grids, the frontiers and the checkpoint files byte-identical to a twin
    without reach jobs."""
    def enqueue(c, is_a, call, t1):
        c.frontier_enqueue(1)
        if is_a:
            c.reach_enqueue(camera(t1 - 1), 0.1, 2, [camera(0)], True, call % 2 == 0)

    def check(a, outs, call, t1, what):
        want = R.reach(outs["state"][0], outs["field"][0], outs["field"][1], 0.1, camera(t1 - 1), 0.1, 2, [camera(0)],
                       outs["shared"]["frontiers"][:2], 64, 1 << 14, 1024)
        same(a.reach_wait(), want, what)

    twin_drive(tmp_path, lambda c: c.frontier_enable(32, 4096), lambda a: a.reach_enable(64, 1 << 14, 1024), enqueue,
               lambda c: {"frontiers": c.frontier_wait()}, check)


def test_rejected_frame_comes_back_from_wait():
    goals = []

    def enqueue(b, first):
        goals.extend([camera(0), camera(first - 1) + 1.0])
        b.reach_enqueue(camera(first - 1), 0.0, 1, goals, False, True)

    r = rejected_known(lambda b: b.reach_enable(8, 1 << 12, 512), enqueue)
    dist, origin, _ = r.field
    e = rejected(r.ctx.reach_wait)
    same(e.reach, R.reach(r.state, dist, origin, r.voxel, camera(r.first - 1), 0.0, 1, goals, None, 8, 1 << 12, 512), "rejected")
    assert e.reach[0]["n_reached"] > 0
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    D3 = ctypes.c_double * 3
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    st = np.full((4, 5, 6), FREE, np.uint8)
    s = D3(0.1, 0.1, 0.1)
    g = np.zeros((2, 3))
    assert lib.dsm_reach_enable(ctx.h, 1, 1, 1) == -7                     # before dsm_field_enable
    ctx.field_enable(0.2, 6, 5, 4)
    assert lib.dsm_reach_enable(ctx.h, 1, 1, 1) == -7                     # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 0, None, 0, 0, 0) == -7   # before dsm_reach_enable
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == -7
    BIG = R.MAX_CAPACITY
    for mt, mp, mr in [(-1, 0, 1), (0, -1, 1), (BIG + 1, 0, 1), (0, BIG + 1, 1), (0, 0, 0), (0, 0, R.MAX_ROUNDS + 1), (0, 0, -1)]:
        assert lib.dsm_reach_enable(ctx.h, mt, mp, mr) == -1, (mt, mp, mr)
    assert lib.dsm_reach_enable(None, 1, 1, 1) == -1
    ctx.reach_enable(2, 8, 64)
    assert lib.dsm_reach_enable(ctx.h, 1, 1, 1) == -7                     # once
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 0, None, 0, 0, 0) == -7   # no field request yet
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == -7        # nothing enqueued
    ctx.field_enqueue((0, 0, 0), 1)                                       # a plain request
    ctx.field_wait()
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 0, None, 0, 0, 0) == -7
    load_known(ctx, st, (0, 0, 0), 0.2)
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 0, None, 0, 1, 0) == -7   # with frontiers, without a frontier job
    nan, inf = float("nan"), float("inf")
    for args in [(D3(nan, 0, 0), 0.0, 0, None, 0), (D3(0, inf, 0), 0.0, 0, None, 0), (s, -0.1, 0, None, 0), (s, nan, 0, None, 0),
                 (s, inf, 0, None, 0), (s, 0.0, -1, None, 0), (s, 0.0, 5, None, 0), (s, 0.0, 0, None, -1), (s, 0.0, 0, None, 3),
                 (s, 0.0, 0, None, 1), (s, 0.0, 0, np.array([[0, nan, 0.0]]).ctypes.data, 1), (None, 0.0, 0, None, 0)]:
        assert lib.dsm_reach_enqueue(ctx.h, *args, 0, 0) == -1, args
    assert lib.dsm_reach_enqueue(None, s, 0.0, 0, None, 0, 0, 0) == -1
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 4, g.ctypes.data, 2, 0, 0) == 0
    assert lib.dsm_reach_enqueue(ctx.h, s, 0.0, 0, None, 0, 0, 0) == -7   # one job in flight
    info = np.zeros(1, capi.REACH_INFO_DTYPE)
    cost = ctypes.c_void_p(1)
    assert lib.dsm_reach_wait(ctx.h, info.ctypes.data, None, None, ctypes.byref(cost)) == 0
    assert cost.value is None                                             # no host copy
    assert info[0]["n_traversable"] == st.size and info[0]["n_reached"] == st.size and info[0]["n_targets"] == 2
    assert lib.dsm_reach_wait(ctx.h, None, None, None, None) == -7
    ctx.close()


# ---- the node ----
def test_node_reach_equals_the_model_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers() and reach(with_frontiers) from
    the camera equal the model over the grids the driver dumps; clouds, PLY and PCD files equal a twin without reach
    jobs; reach() without a frontiers() call on the frame, and after load_state until the next fused frame, returns
    DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("reach_main", str(tmp_path), cam, sc, node_args() + [64, 1 << 16, 2048, RELOAD], tag="a", after=[pa])
    q = run_driver("reach_main", str(tmp_path), cam, sc, node_args() + [0, 0, 0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, k = r.i(), r.i()
        start = r.take(np.float64, 3).copy()
        radius = float(r.take(np.float32, 1)[0])
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        info = r.take(np.uint8, R.INFO_DTYPE.itemsize).view(R.INFO_DTYPE)[0].copy()
        targets, path = r.lst(R.TARGET_DTYPE), r.lst(np.int32)
        before, after_load = r.i(), r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        want = R.reach(state, dist, origin, voxel, start, radius, k, (), (clusters, vox), 64, 1 << 16, 2048)
        same((info, targets, path, None), want, f"message {t}")
        found += int((targets["status"] == 0).sum()) > 0
        assert before == -7, f"message {t}: reach() before frontiers()"
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: reach() after load_state"
    assert found > 0
    twin_node_tail(r, q, pa, pb)
