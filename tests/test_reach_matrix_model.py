"""The matrix model of oracle/pyoracle_reach_matrix (DESIGN.md §8.13) on the CPU: a converged matrix against scipy's Dijkstra
and its metric properties; every row against the round emulator started at that site, unconverged rows included;
scheduling on active tiles only against dense scheduling; the active-tile count and the capacity cut by hand; the snap
of voxel centres, sites outside the grid, blocked, repeated and sharing a tile; and the refusals the library makes
without a device."""
import ctypes

import numpy as np
import pytest
from scipy.sparse import csgraph

import pyoracle_reach as R
import pyoracle_reach_matrix as RM
from densesurfelmapping_b200 import capi
from test_frontier_model import serpentine

FREE, UNKNOWN, OCCUPIED = R.FREE, R.UNKNOWN, R.OCCUPIED


def centre(c, origin, voxel):
    """The world centre ((o + x) + 0.5) v of voxel c, in fp64 from the fp32 edge."""
    v = float(np.float32(voxel))
    return tuple((float(origin[k] + c[k]) + 0.5) * v for k in range(3))


def random_grid(shape_xyz, p, seed):
    rng = np.random.default_rng(seed)
    st = rng.choice(3, size=shape_xyz[::-1], p=p).astype(np.uint8)
    return st, np.full(st.shape, np.inf, np.float32), rng


def traversable_sites(trav, rng, n):
    idx = np.flatnonzero(trav.reshape(-1))
    return rng.choice(idx, size=min(n, len(idx)), replace=False)


def xyz(u, shape_zyx):
    nz, ny, nx = shape_zyx
    return (u % nx, u // nx % ny, u // (nx * ny))


def sparse_emulate(trav, u, max_rounds):
    """The round rule run as the device's matrix job runs it: only active tiles are ever scheduled.  Returns (cost,
    rounds, converged); it must equal R.emulate on the dense grid."""
    nz, ny, nx = trav.shape
    act = RM.active_tiles(trav)
    tn = act.shape[::-1]
    big = np.int64(R.INF)
    P = [tn[2] * R.TILE + 2, tn[1] * R.TILE + 2, tn[0] * R.TILE + 2]
    C = np.full(P, big, np.int64)
    T = np.zeros(P, bool)
    T[1:nz + 1, 1:ny + 1, 1:nx + 1] = trav
    if u < 0:
        return np.full(trav.shape, R.INF, np.uint32), 0, 1
    ux, uy, uz = xyz(u, trav.shape)
    C[uz + 1, uy + 1, ux + 1] = 0
    sched, rounds = {(ux // R.TILE, uy // R.TILE, uz // R.TILE)}, 0
    for _ in range(max_rounds):
        if not sched:
            break
        assert all(act[c, b, a] for a, b, c in sched), "an inactive tile was scheduled"
        rounds += 1
        new_sched = set()
        staged = {}
        for (tx, ty, tz) in sorted(sched):
            z0, y0, x0 = tz * R.TILE, ty * R.TILE, tx * R.TILE
            B = C[z0:z0 + R.TILE + 2, y0:y0 + R.TILE + 2, x0:x0 + R.TILE + 2].copy()
            M = T[z0 + 1:z0 + R.TILE + 1, y0 + 1:y0 + R.TILE + 1, x0 + 1:x0 + R.TILE + 1]
            B0 = B[1:-1, 1:-1, 1:-1].copy()
            while True:
                best = B[1:-1, 1:-1, 1:-1].copy()
                for dx, dy, dz in R.MOVES:
                    nb = B[1 + dz:R.TILE + 1 + dz, 1 + dy:R.TILE + 1 + dy, 1 + dx:R.TILE + 1 + dx]
                    np.minimum(best, np.where(nb < big, nb + int(R.chamfer(dx, dy, dz)), big), out=best)
                new = np.where(M, best, B[1:-1, 1:-1, 1:-1])
                if (new == B[1:-1, 1:-1, 1:-1]).all():
                    break
                B[1:-1, 1:-1, 1:-1] = new
            staged[(tx, ty, tz)] = B[1:-1, 1:-1, 1:-1]
            if rounds == 1 or (B[1:-1, 1:-1, 1:-1] != B0).any():
                for dz in (-1, 0, 1):
                    for dy in (-1, 0, 1):
                        for dx in (-1, 0, 1):
                            a, b, c = tx + dx, ty + dy, tz + dz
                            if 0 <= a < tn[0] and 0 <= b < tn[1] and 0 <= c < tn[2] and act[c, b, a]:
                                new_sched.add((a, b, c))
        for (tx, ty, tz), V in staged.items():
            C[tz * R.TILE + 1:tz * R.TILE + R.TILE + 1, ty * R.TILE + 1:ty * R.TILE + R.TILE + 1, tx * R.TILE + 1:tx * R.TILE + R.TILE + 1] = V
        sched = new_sched
    return C[1:nz + 1, 1:ny + 1, 1:nx + 1].astype(np.uint32), rounds, int(not sched)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_converged_matrix_equals_dijkstra_and_is_a_metric(seed):
    shape, o, v = (21, 18, 11), (-7, 3, -2), 0.25
    st, dist, rng = random_grid(shape, (0.1, 0.15, 0.75), seed)
    trav = R.traversable(st, dist, 0.0)
    u = traversable_sites(trav, rng, 12)
    pts = [centre(xyz(int(x), st.shape), o, v) for x in u]
    info, sites, M = RM.matrix(st, dist, o, v, pts, 0.0, 0, max_tiles=1 << 20)
    assert info["status"] == 0 and (sites["status"] == 0).all() and (sites["converged"] == 1).all()
    assert sites["voxel"].tolist() == u.tolist()
    d = csgraph.dijkstra(R.graph(trav), directed=False, indices=u)[:, u]
    want = np.where(np.isfinite(d), d, R.INF).astype(np.uint32)
    assert M.tobytes() == want.tobytes()
    assert (np.diag(M) == 0).all() and (M == M.T).all()
    fin = M.astype(np.int64)
    fin[M == R.INF] = 1 << 40
    for k in range(len(u)):   # the triangle inequality through every site k
        assert (fin <= fin[:, k:k + 1] + fin[k:k + 1, :]).all(), k


@pytest.mark.parametrize("rounds", [1, 7, 40, 4096])
def test_rows_equal_the_emulator_unconverged_serpentine_included(rounds):
    st = serpentine(48, 40, 8)
    dist = np.full(st.shape, np.inf, np.float32)
    trav = R.traversable(st, dist, 0.0)
    rng = np.random.default_rng(rounds)
    u = traversable_sites(trav, rng, 6)
    pts = [centre(xyz(int(x), st.shape), (0, 0, 0), 0.2) for x in u] + [(-1.0, 0.0, 0.0)]
    info, sites, M = RM.matrix(st, dist, (0, 0, 0), 0.2, pts, 0.0, 1, max_tiles=1 << 20, max_rounds=rounds)
    assert info["status"] == 0 and info["n_active_tiles"] == RM.active_tiles(trav).sum()
    assert info["rounds"] == sites["rounds"].max()
    for i, x in enumerate(u):
        cost, r, conv = R.emulate(trav, int(x), rounds)
        assert (sites[i]["rounds"], sites[i]["converged"], sites[i]["n_reached"]) == (r, conv, int((cost != R.INF).sum()))
        assert M[i, :len(u)].tobytes() == cost.reshape(-1)[u].tobytes()
        exact = R.dijkstra(trav, int(x)).reshape(-1)[u]
        assert (M[i, :len(u)] >= exact).all()
    assert rounds == 4096 or (sites["converged"][:len(u)] == 0).any()
    assert sites[-1]["status"] == 1 and sites[-1]["voxel"] == -1 and (M[-1] == R.INF).all() and (M[:, -1] == R.INF).all()
    assert (sites[-1]["rounds"], sites[-1]["converged"], sites[-1]["n_reached"]) == (0, 1, 0)


@pytest.mark.parametrize("case", range(6))
def test_active_tile_scheduling_equals_dense_scheduling(case):
    shapes = [(20, 17, 9), (33, 9, 1), (1, 1, 40), (24, 24, 24), (48, 40, 8), (16, 16, 16)]
    shape = shapes[case]
    if case == 4:
        st = serpentine(*shape)
    elif case == 5:   # a start walled off in its tile, whose neighbours are partly inactive
        st = np.full(shape[::-1], OCCUPIED, np.uint8)
        st[8:, :, :] = FREE
        st[:8, :8, :8] = OCCUPIED
        st[7, 7, 7] = FREE
    else:
        st = random_grid(shape, (0.3, 0.3, 0.4), case)[0]
    trav = R.traversable(st, np.full(st.shape, np.inf, np.float32), 0.0)
    rng = np.random.default_rng(case)
    starts = list(traversable_sites(trav, rng, 3)) + ([7 * 16 * 16 + 7 * 16 + 7] if case == 5 else [])
    for u in starts:
        for rounds in (1, 3, 10, 4096):
            want = R.emulate(trav, int(u), rounds)
            got = sparse_emulate(trav, int(u), rounds)
            assert got[0].tobytes() == want[0].tobytes() and got[1:] == want[1:], (shape, u, rounds)


def test_active_tile_count_by_hand():
    # 9 x 17 x 3: tiles 2 x 3 x 1; mark voxels in three tiles, one of them the clipped corner tile
    st = np.full((3, 17, 9), OCCUPIED, np.uint8)
    st[0, 0, 0] = FREE          # tile (0, 0, 0)
    st[2, 16, 8] = FREE         # tile (1, 2, 0), one voxel wide on x and y
    st[1, 9, 3] = FREE          # tile (0, 1, 0)
    st[1, 10, 4] = FREE         # the same tile again
    trav = R.traversable(st, np.full(st.shape, np.inf, np.float32), 0.0)
    act = RM.active_tiles(trav)
    assert act.shape == (1, 3, 2) and act.sum() == 3
    assert act[0, 0, 0] and act[0, 2, 1] and act[0, 1, 0] and not act[0, 0, 1]
    for shape_zyx, want in [((1, 1, 1), 1), ((1, 1, 17), 3), ((1, 9, 1), 2), ((13, 1, 1), 2)]:
        st = np.full(shape_zyx, FREE, np.uint8)
        assert RM.active_tiles(R.traversable(st, np.full(shape_zyx, np.inf, np.float32), 0.0)).sum() == want, shape_zyx
    # the radius decides: a grid whose distances fall short of it has no active tile
    st = np.full((5, 6, 7), FREE, np.uint8)
    info, sites, M = RM.matrix(st, np.full(st.shape, 0.1, np.float32), (0, 0, 0), 0.2, [(0.1, 0.1, 0.1)], 0.2, 4, max_tiles=1)
    assert info["n_active_tiles"] == 0 and info["n_traversable"] == 0 and info["status"] == 0 and sites[0]["status"] == 2


def test_the_capacity_cut():
    st, dist, rng = random_grid((30, 20, 12), (0.2, 0.2, 0.6), 5)
    trav = R.traversable(st, dist, 0.0)
    n_active = int(RM.active_tiles(trav).sum())
    assert n_active == 4 * 3 * 2
    pts = [centre(xyz(int(x), st.shape), (0, 0, 0), 0.2) for x in traversable_sites(trav, rng, 5)]
    ok = RM.matrix(st, dist, (0, 0, 0), 0.2, pts, 0.0, 0, max_tiles=n_active)
    cut = RM.matrix(st, dist, (0, 0, 0), 0.2, pts, 0.0, 0, max_tiles=n_active - 1)
    assert ok[0]["status"] == 0 and (ok[2] != R.INF).any() and ok[0]["rounds"] > 0
    assert cut[0]["status"] == 1 and cut[0]["n_active_tiles"] == n_active and cut[0]["rounds"] == 0
    assert (cut[2] == R.INF).all()
    for f in ("voxel", "status", "approach"):
        assert cut[1][f].tolist() == ok[1][f].tolist(), f
    assert (cut[1]["rounds"] == 0).all() and (cut[1]["converged"] == 0).all() and (cut[1]["n_reached"] == 0).all()


@pytest.mark.parametrize("voxel", [0.05, 0.1, 0.2, 0.3, 0.125, 1.7])
def test_voxel_centres_snap_to_themselves(voxel):
    shape = (9, 10, 11)
    rng = np.random.default_rng(int(voxel * 1000))
    for o in [(0, 0, 0), (-5, 7, -3), (1 << 24, -(1 << 24), (1 << 24) - 9), (-(1 << 24) + 3, (1 << 23) + 1, 12345)]:
        for c in rng.integers(0, shape, size=(30, 3)).tolist() + [[0, 0, 0], [8, 9, 10]]:
            assert R.voxel_of(centre(c, o, voxel), o, voxel, shape) == tuple(c), (voxel, o, c)


def test_outside_blocked_repeated_and_shared_tile_sites():
    st = np.full((6, 12, 12), FREE, np.uint8)
    st[:, :, 6] = OCCUPIED             # a wall at x = 6 ...
    st[:, 11, 6] = FREE                # ... with a gap at y = 11
    st[3, 3, 9] = OCCUPIED
    dist = np.full(st.shape, np.inf, np.float32)
    o, v = (2, -3, 0), 0.5
    pts = [centre((1, 1, 1), o, v), centre((2, 1, 1), o, v),     # two sites in one tile
           centre((9, 3, 3), o, v),                               # an occupied voxel: snapped within the window
           centre((1, 1, 1), o, v),                               # a repeat
           centre((20, 0, 0), o, v),                              # outside the grid
           centre((10, 2, 2), o, v)]
    info, sites, M = RM.matrix(st, dist, o, v, pts, 0.0, 1, max_tiles=1 << 10)
    assert sites["status"].tolist() == [0, 0, 0, 0, 1, 0]
    assert sites[2]["approach"] == 10 and sites[2]["voxel"] != (3 * 12 + 3) * 12 + 9
    assert M[0].tobytes() == M[3].tobytes() and M[0, 3] == 0 and M[3, 0] == 0 and M[0, 1] == 10
    assert (M[4] == R.INF).all() and (M[:, 4] == R.INF).all()
    assert M[0, 5] > 10 * 9   # around the wall through the gap
    info, sites, M = RM.matrix(st, dist, o, v, pts, 0.0, 0, max_tiles=1 << 10)
    assert sites[2]["status"] == 2 and sites[2]["voxel"] == -1 and (M[2] == R.INF).all() and (M[:, 2] == R.INF).all()
    assert (sites[2]["rounds"], sites[2]["converged"], sites[2]["n_reached"]) == (0, 1, 0)


def test_calls_are_declared_and_refuse_a_null_context():
    lib = capi.load_library()
    for name in ["dsm_reach_matrix_enable", "dsm_reach_matrix_enqueue", "dsm_reach_matrix_wait"]:
        assert name in capi.EXPORTS and hasattr(lib, name)
    pts = np.zeros((1, 3))
    assert lib.dsm_reach_matrix_enable(None, 1, 1, 1) == -1
    assert lib.dsm_reach_matrix_enqueue(None, pts.ctypes.data, 1, 0.0, 0) == -1
    assert lib.dsm_reach_matrix_wait(None, None, None, None) == -1
    assert capi.REACH_SITE_DTYPE == RM.SITE_DTYPE and capi.REACH_MATRIX_INFO_DTYPE == RM.MATRIX_INFO_DTYPE
    assert RM.SITE_DTYPE.itemsize == 32 and RM.MATRIX_INFO_DTYPE.itemsize == 64
    assert ctypes.sizeof(ctypes.c_int32) * 16 == RM.MATRIX_INFO_DTYPE.itemsize
