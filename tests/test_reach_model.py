"""The reach model of oracle/pyoracle_reach (DESIGN.md §8.11) on the CPU: the chamfer weights, scipy's Dijkstra against a
plain heapq Dijkstra, the tile-round emulator against Dijkstra (and a round count counted by hand), unconverged jobs,
hand cases of every rule of the definition, both capacity cuts, and the refusals the library makes without a device."""
import ctypes
import heapq

import numpy as np
import pytest

import pyoracle_frontier
import pyoracle_reach as R
from densesurfelmapping_b200 import capi

FREE, UNKNOWN, OCCUPIED = R.FREE, R.UNKNOWN, R.OCCUPIED


def heap_dijkstra(trav, u):
    nz, ny, nx = trav.shape
    cost = np.full(trav.size, R.INF, np.int64)
    cost[u] = 0
    q = [(0, u)]
    while q:
        c, x = heapq.heappop(q)
        if c != cost[x]:
            continue
        px, py, pz = x % nx, x // nx % ny, x // (nx * ny)
        for dx, dy, dz in R.MOVES:
            a, b, d = px + dx, py + dy, pz + dz
            if 0 <= a < nx and 0 <= b < ny and 0 <= d < nz and trav[d, b, a]:
                p = (d * ny + b) * nx + a
                w = c + int(R.chamfer(dx, dy, dz))
                if w < cost[p]:
                    cost[p] = w
                    heapq.heappush(q, (w, p))
    return cost.reshape(trav.shape).astype(np.uint32)


def free_grid(shape_zyx, dist=np.inf):
    return np.full(shape_zyx, FREE, np.uint8), np.full(shape_zyx, dist, np.float32)


def centre(c, origin=(0, 0, 0), voxel=0.5):
    """A world point inside voxel c (x, y, z) of a grid at `origin`."""
    return tuple((c[k] + origin[k] + 0.5) * voxel for k in range(3))


def test_chamfer_closed_form_and_band():
    trav = np.ones((9, 11, 13), bool)
    u = (4 * 11 + 5) * 13 + 6
    cost = R.dijkstra(trav, u)
    z, y, x = np.indices(trav.shape)
    want = R.chamfer(x - 6, y - 5, z - 4)
    assert (cost == want).all()
    d = np.sqrt((x - 6.0) ** 2 + (y - 5.0) ** 2 + (z - 4.0) ** 2) * 10
    m = d > 0
    ratio = want[m] / d[m]
    assert ratio.min() >= 0.98 and ratio.max() <= 1.12, (ratio.min(), ratio.max())
    assert [int(R.chamfer(*m)) for m in [(1, 0, 0), (1, 1, 0), (1, 1, 1)]] == [10, 14, 17]


@pytest.mark.parametrize("seed", range(6))
def test_scipy_equals_heapq_dijkstra(seed):
    rng = np.random.default_rng(seed)
    shape = tuple(rng.integers(3, 12, size=3))
    trav = rng.random(shape) < (0.35 + 0.1 * seed)
    trav.reshape(-1)[0] = True
    assert (R.dijkstra(trav, 0) == heap_dijkstra(trav, 0)).all()


@pytest.mark.parametrize("seed", range(4))
def test_emulator_at_a_generous_cap_equals_dijkstra(seed):
    rng = np.random.default_rng(100 + seed)
    shape = (int(rng.integers(5, 20)), int(rng.integers(5, 30)), int(rng.integers(5, 30)))
    trav = rng.random(shape) < 0.6
    u = int(np.flatnonzero(trav.reshape(-1))[len(np.flatnonzero(trav)) // 2])
    cost, rounds, conv = R.emulate(trav, u, R.MAX_ROUNDS)
    assert conv == 1 and rounds >= 1
    assert (cost == R.dijkstra(trav, u)).all()


def walled_off(shape_zyx, p, density, seed):
    """A random grid of the given traversable density in which p is the only traversable voxel of its 8x8x8 tile."""
    trav = np.random.default_rng(seed).random(shape_zyx) < density
    z, y, x = (slice(c // R.TILE * R.TILE, c // R.TILE * R.TILE + R.TILE) for c in p)
    trav[z, y, x] = False
    trav[p] = True
    return trav


@pytest.mark.parametrize("seed", range(8))
def test_a_start_walled_off_in_its_tile_equals_dijkstra(seed):
    """The start is the only traversable voxel of its tile, on a tile face, edge or corner: it reaches the grid only
    across its tile's faces, so round 0 must schedule the neighbour tiles although it changes nothing."""
    rng = np.random.default_rng(200 + seed)
    shape = tuple(int(n) for n in rng.integers(9, 26, size=3))
    p = tuple(int(rng.choice([7, 8, min(15, n - 1)]) if a < 1 + seed % 3 else rng.integers(0, n)) for a, n in enumerate(shape))
    trav = walled_off(shape, p, 0.75, seed)
    u = (p[0] * shape[1] + p[1]) * shape[2] + p[2]
    want = R.dijkstra(trav, u)
    cost, rounds, conv = R.emulate(trav, u, R.MAX_ROUNDS)
    assert conv == 1 and rounds >= 2
    assert (cost == want).all(), f"{int((cost != want).sum())} costs differ"
    assert (want != R.INF).sum() > 1


def test_walled_off_starts_by_hand():
    """A row of 20 voxels from x = 7 with x < 7 blocked: round 0 reaches nothing beyond the start, yet schedules tiles 0
    and 1; round 1 fills tile 1, round 2 tile 2, round 3 changes nothing.  And a 16^3 free grid whose inner octant is
    occupied but for its corner (7, 7, 7), the start: everything free is reached, at Dijkstra's costs."""
    trav = np.ones((1, 1, 20), bool)
    trav[0, 0, :7] = False
    cost, rounds, conv = R.emulate(trav, 7, 100)
    assert (rounds, conv) == (4, 1)
    assert (cost.ravel()[7:] == 10 * np.arange(13)).all() and (cost.ravel()[:7] == R.INF).all()
    st, dist = free_grid((16, 16, 16))
    st[:8, :8, :8] = OCCUPIED
    st[7, 7, 7] = FREE
    info, recs, path, cost = R.reach(st, dist, (0, 0, 0), 0.5, centre((7, 7, 7)), 0.0, 0, [centre((15, 15, 15))])
    trav = R.traversable(st, dist, 0.0)
    assert info["converged"] == 1 and info["n_reached"] == info["n_traversable"] == 16 ** 3 - 8 ** 3 + 1
    assert (cost == R.dijkstra(trav, int(info["start_voxel"]))).all()
    assert recs[0]["status"] == 0 and recs[0]["cost"] == 8 * 17


def test_round_count_by_hand():
    """A row of 20 free voxels from x = 0: tiles [0, 8), [8, 16), [16, 20).  Round 0 fills tile 0; round 1 tile 1 (tile 0
    unchanged); round 2 tile 2; round 3 changes nothing: 4 rounds, converged.  Capped at 2 rounds, tile 2 is unreached."""
    trav = np.ones((1, 1, 20), bool)
    cost, rounds, conv = R.emulate(trav, 0, 100)
    assert (rounds, conv) == (4, 1) and (cost.ravel() == 10 * np.arange(20)).all()
    cost, rounds, conv = R.emulate(trav, 0, 2)
    assert (rounds, conv) == (2, 0)
    assert (cost.ravel()[:16] == 10 * np.arange(16)).all() and (cost.ravel()[16:] == R.INF).all()
    cost, rounds, conv = R.emulate(trav, 0, 3)
    assert (rounds, conv) == (3, 0) and (cost.ravel() == 10 * np.arange(20)).all()   # exact, not yet known to be


def serpentine_grid(nx, ny, nz):
    """Walls across y every other row with a gap alternating at either end: one long corridor."""
    st = np.full((nz, ny, nx), FREE, np.uint8)
    for y in range(1, ny, 2):
        st[:, y, :] = OCCUPIED
        gap = nx - 1 if (y // 2) % 2 == 0 else 0
        st[:, y, gap] = FREE
    return st


def test_unconverged_is_an_upper_bound_and_paths_stay_under_it():
    st = serpentine_grid(24, 23, 2)
    dist = np.full(st.shape, np.inf, np.float32)
    goals = [centre((x, y, 1)) for x, y in [(3, 22), (20, 12), (0, 6), (23, 0)]]
    for cap in (1, 3, 7, 20):
        info, recs, path, cost = R.reach(st, dist, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 0, goals, max_rounds=cap)
        exact = R.dijkstra(R.traversable(st, dist, 0.0), int(info["start_voxel"]))
        assert info["converged"] == 0 and info["rounds"] == cap
        assert (cost >= exact).all()
        trav = R.traversable(st, dist, 0.0)
        nz, ny, nx = st.shape
        for r in recs[recs["status"] == 0]:
            p = path[r["path_offset"]:r["path_offset"] + r["path_len"]]
            assert p[0] == info["start_voxel"] and p[-1] == r["viewpoint"]
            xyz = np.stack([p % nx, p // nx % ny, p // (nx * ny)], 1)
            step = np.diff(xyz, axis=0)
            assert (np.abs(step).max(axis=1) == 1).all() and trav.reshape(-1)[p].all()
            w = int(R.chamfer(step[:, 0], step[:, 1], step[:, 2]).sum())
            assert exact.reshape(-1)[r["viewpoint"]] <= w <= cost.reshape(-1)[r["viewpoint"]]
    info, recs, path, cost = R.reach(st, dist, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 0, goals)
    assert info["converged"] == 1 and (recs["status"] == 0).all()


def test_radius_at_a_stored_distance_and_radius_zero():
    st, dist = free_grid((1, 1, 6))
    dist[0, 0, :] = np.float32([0.5, 1.0, 1.5, 1.0, 0.5, 0.25])
    for radius, want in [(1.0, [0, 1, 1, 1, 0, 0]), (np.float32(1.0) + np.float32(1e-7), [0, 0, 1, 0, 0, 0]), (0.0, [1] * 6)]:
        assert R.traversable(st, dist, radius).ravel().astype(int).tolist() == want
    st[0, 0, 5] = OCCUPIED
    dist[0, 0, 5] = 0.0
    assert not R.traversable(st, dist, 0.0).ravel()[5]   # radius 0 still needs a free voxel


def test_start_outside_blocked_and_snapped():
    st, dist = free_grid((3, 4, 5))
    st[:] = OCCUPIED
    st[2, 3, 4] = FREE
    o = (-2, 3, 1)
    u = (2 * 4 + 3) * 5 + 4
    for p, k, want in [((-100.0, 0.0, 0.0), 4, (-1, 1, 0)),                 # outside
                       (centre((0, 0, 0), o), 1, (-1, 2, 0)),                # blocked: nothing traversable in the window
                       (centre((0, 0, 0), o), 4, (u, 0, 58)),                # the window of 4 reaches (4, 3, 2)
                       (centre((3, 2, 1), o), 1, (u, 0, 17)),
                       (centre((4, 3, 2), o), 0, (u, 0, 0))]:
        info, recs, path, cost = R.reach(st, dist, o, 0.5, p, 0.0, k)
        assert (int(info["start_voxel"]), int(info["start_status"]), int(info["start_approach"])) == want, (p, k)
        assert info["n_reached"] == (1 if want[1] == 0 else 0)
        # one tile: round 0 (the seed) schedules it again, round 1 changes nothing
        assert info["rounds"] == (2 if want[1] == 0 else 0) and info["converged"] == 1


def test_ties_in_the_snap_the_viewpoint_the_member_and_the_predecessor():
    st, dist = free_grid((3, 3, 3))
    st[1, 1, 1] = OCCUPIED                       # the centre: every face neighbour ties at chamfer 10
    s = centre((1, 1, 1))
    info, _, _, _ = R.reach(st, dist, (0, 0, 0), 0.5, s, 0.0, 1)
    assert info["start_voxel"] == (0 * 3 + 1) * 3 + 1 and info["start_approach"] == 10   # (1, 1, 0): the lowest index
    # a goal at the blocked centre: six face neighbours at window cost cost[u] + 10; the lowest total, then index, wins
    info, recs, path, cost = R.reach(st, dist, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 1, [s])
    flat = cost.reshape(-1).astype(np.int64)
    idx = [(z * 3 + y) * 3 + x for x, y, z in [(0, 1, 1), (2, 1, 1), (1, 0, 1), (1, 2, 1), (1, 1, 0), (1, 1, 2)]]
    idx += [(z * 3 + y) * 3 + x for z in range(3) for y in range(3) for x in range(3) if (x, y, z) != (1, 1, 1)]
    keys = sorted((int(flat[i]) + int(R.chamfer(i % 3 - 1, i // 3 % 3 - 1, i // 9 - 1)), i) for i in set(idx))
    assert (int(recs[0]["cost"]), int(recs[0]["viewpoint"])) == keys[0]
    # the predecessor: from (2, 2, 0) back to (0, 0, 0) in a 3x3x1 free grid, many tight paths; the lowest index is taken
    st2, d2 = free_grid((1, 3, 3))
    info, recs, path, cost = R.reach(st2, d2, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 0, [centre((2, 2, 0))])
    assert path.tolist() == [0, 4, 8] and recs[0]["cost"] == 28
    info, recs, path, cost = R.reach(st2, d2, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 0, [centre((2, 1, 0))])
    assert recs[0]["cost"] == 24 and path.tolist() == [0, 1, 5]   # (1,0) + edge and (1,1) + face tie at 10; 1 < 4
    # the member: members 1 and 3 too close to the unknown ends to be traversable; both see the start (2) at cost 10
    st3, d3 = free_grid((1, 1, 5))
    st3[0, 0, [0, 4]] = UNKNOWN
    d3[0, 0, :] = [0.0, 0.5, 1.0, 0.5, 0.0]
    cl = np.zeros(1, pyoracle_frontier.CLUSTER_DTYPE)
    cl["n_voxels"], cl["first"], cl["offset"] = 2, 1, 0
    for members in ([1, 3], [3]):
        cl["n_voxels"], cl["first"] = len(members), members[0]
        info, recs, path, cost = R.reach(st3, d3, (0, 0, 0), 0.5, centre((2, 0, 0)), 1.0, 1, frontier=(cl, np.int32(members)))
        assert (recs[0]["target"], recs[0]["viewpoint"], recs[0]["cost"], recs[0]["approach"]) == (members[0], 2, 10, 10)


def test_window_clipping_and_unreachable_goals():
    st, dist = free_grid((4, 4, 4))
    st[:, :, 2] = OCCUPIED                              # a wall at x = 2: x = 3 is unreachable from x = 0
    info, recs, path, cost = R.reach(st, dist, (0, 0, 0), 0.5, centre((0, 0, 0)), 0.0, 1,
                                     [centre((3, 3, 3)), centre((-1, 0, 0)), centre((2, 3, 3)), centre((0, 0, 0))])
    assert recs["status"].tolist() == [2, 1, 0, 0]
    assert recs["target"].tolist() == [63, -1, (3 * 4 + 3) * 4 + 2, 0]
    # (1, 2, 2) at 31 + 17 beats (1, 3, 3), (1, 2, 3) and (1, 3, 2) at 45 + 10, 41 + 14 and 41 + 14
    assert recs[2]["viewpoint"] == (2 * 4 + 2) * 4 + 1 and recs[2]["approach"] == 17 and recs[2]["cost"] == 48
    assert recs[3]["cost"] == 0 and recs[3]["path_len"] == 1
    assert recs[0]["cost"] == R.INF and recs[0]["viewpoint"] == -1 and recs[0]["path_offset"] == -1
    assert info["n_targets"] == 4 and info["n_path_voxels"] == recs[2]["path_len"] + 1
    # the corner goal's window is clipped to 2x2x2 voxels
    x, y, z, *_ = R.window((0, 0, 0), 1, (4, 4, 4))
    assert len(x) == 8


def test_clusters_offset_minus_one_and_both_capacity_cuts():
    st, dist = free_grid((2, 6, 12))
    st[:, 0, 3] = UNKNOWN
    st[:, 5, 9] = UNKNOWN
    st[:, 3, 6] = UNKNOWN
    fc, fv, _ = pyoracle_frontier.frontiers(st, (0, 0, 0), 0.5, 1, 8, 1 << 10)
    assert len(fc) >= 2
    start = centre((0, 2, 0))
    goals = [centre((11, 5, 1)), centre((0, 0, 0))]
    full = R.reach(st, dist, (0, 0, 0), 0.5, start, 0.0, 1, goals, (fc, fv), max_targets=16, max_path=1 << 10)
    assert (full[1]["status"] == 0).all() and full[0]["n_clusters_total"] == len(fc)
    cut = fc.copy()
    cut["offset"][1:] = -1                             # the frontier list held the first cluster only
    r = R.reach(st, dist, (0, 0, 0), 0.5, start, 0.0, 1, goals, (cut, fv[:fc[0]["n_voxels"]]), max_targets=16)
    assert r[1]["status"].tolist() == [0, 0, 0] + [3] * (len(fc) - 1)
    assert (r[1]["target"][3:] == fc["first"][1:]).all()
    r = R.reach(st, dist, (0, 0, 0), 0.5, start, 0.0, 1, goals, (fc, fv), max_targets=3)   # one cluster kept
    assert r[0]["n_targets"] == 3 and r[0]["n_clusters_total"] == len(fc) and r[1].tobytes() == full[1][:3].tobytes()
    lens = full[1]["path_len"]
    for cap in (0, int(lens[0]), int(lens[0] + lens[1]) - 1):
        r = R.reach(st, dist, (0, 0, 0), 0.5, start, 0.0, 1, goals, (fc, fv), max_targets=16, max_path=cap)
        listed = np.cumsum(lens) <= cap
        assert (r[1]["path_offset"] >= 0).tolist() == listed.tolist()
        assert r[0]["n_path_voxels"] == int(lens[listed].sum()) and len(r[2]) == r[0]["n_path_voxels"]
        assert (r[1]["path_len"] == lens).all()


def test_calls_are_declared_and_refuse_a_null_context():
    lib = capi.load_library()
    for name in ["dsm_reach_enable", "dsm_reach_enqueue", "dsm_reach_wait"]:
        assert name in capi.EXPORTS and hasattr(lib, name), name
    start = (ctypes.c_double * 3)(0, 0, 0)
    assert lib.dsm_reach_enable(None, 1, 1, 1) == -1
    assert lib.dsm_reach_enqueue(None, start, 0.0, 0, None, 0, 0, 0) == -1
    assert lib.dsm_reach_wait(None, None, None, None, None) == -1
    assert capi.REACH_TARGET_DTYPE.itemsize == 32 and capi.REACH_INFO_DTYPE.itemsize == 64
    assert capi.REACH_TARGET_DTYPE == R.TARGET_DTYPE and capi.REACH_INFO_DTYPE == R.INFO_DTYPE
