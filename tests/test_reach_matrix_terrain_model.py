"""The terrain matrix model of oracle/pyoracle_reach_matrix_terrain (DESIGN.md §8.22) on the CPU: a converged matrix
against scipy's Dijkstra on the 8-connected 10/14 graph for all six up axes, with its metric properties; every row
against the terrain reach model from that site, unconverged rows included; flat scheduling on active tiles only against
dense scheduling; flat active-tile counts by hand and both sides of the capacity cut; cell centres at any height
snapping to themselves; sites outside, above, below, blocked, repeated and sharing a tile; and every refusal."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

import pyoracle_field_known
import pyoracle_reach as R
import pyoracle_reach_matrix as RM
import pyoracle_reach_matrix_terrain as RMT
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR
from densesurfelmapping_b200 import capi

FREE, OCCUPIED, UNKNOWN = R.FREE, R.OCCUPIED, R.UNKNOWN
BIG_TILES = 1 << 10


def scene(rng, shape, up, p_box=0.12, p_hole=0.05):
    """A state grid [nz][ny][nx] with a flat ground along `up`, boxes three voxels high and holes without support."""
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


def plane(status, voxel=0.1, origin=(0, 0, 0), n_up=4):
    """A terrain job's result (up = +3) with the status plane [Q][P], and the field grid (P, Q, n_up) it came from."""
    st = np.asarray(status, np.uint8)[None]
    clear, _, _ = pyoracle_field_known.state_field(st, voxel)
    info = np.zeros(1, TR.INFO_DTYPE)[0]
    info["origin"], info["m"], info["up"] = origin, (st.shape[2], st.shape[1], 1), 3
    return (info, None, st, None, clear), (st.shape[2], st.shape[1], n_up)


def centre(p, q, voxel=0.1, origin=(0, 0, 0), z=0.0):
    v = float(np.float32(voxel))
    return ((p + origin[0] + 0.5) * v, (q + origin[1] + 0.5) * v, z)


def serpentine(Q, P):
    st = np.full((Q, P), FREE, np.uint8)
    for i, q in enumerate(range(3, Q - 1, 4)):
        st[q, :] = OCCUPIED
        st[q, P - 1 if i % 2 == 0 else 0] = FREE
    return st


def dijkstra8(trav, starts):
    """float [len(starts)][Q P]: the exact costs over the 8-connected 10/14 graph of trav [Q][P], restated."""
    Q, P = trav.shape
    rows, cols, w = [], [], []
    q, p = np.nonzero(trav)
    for dq, dp, c in ((0, 1, 10), (1, 0, 10), (1, 1, 14), (1, -1, 14)):
        a, b = q + dq, p + dp
        m = (a < Q) & (b >= 0) & (b < P)
        m[m] = trav[a[m], b[m]]
        rows.append(q[m] * P + p[m])
        cols.append(a[m] * P + b[m])
        w.append(np.full(int(m.sum()), c, np.float64))
    g = sparse.csr_matrix((np.concatenate(w), (np.concatenate(rows), np.concatenate(cols))), shape=(trav.size, trav.size))
    return csgraph.dijkstra(g, directed=False, indices=starts)


def trav_of(terrain, radius=0.0):
    return RMT.plane(terrain, radius)[0]


def sparse_flat_emulate(trav, u, max_rounds):
    """The flat round rule run as the device's matrix job runs it: only active flat tiles are ever scheduled.  Returns
    (cost [Q][P], rounds, converged); it must equal pyoracle_reach_terrain.emulate, which schedules every tile."""
    Q, P = trav.shape
    act = RMT.active_tiles(trav)
    tq, tp = act.shape
    TX, TY = RT.TX, RT.TY
    big = np.int64(R.INF)
    C = np.full((tq * TY + 2, tp * TX + 2), big, np.int64)
    T = np.zeros(C.shape, bool)
    T[1:Q + 1, 1:P + 1] = trav
    if u < 0:
        return np.full(trav.shape, R.INF, np.uint32), 0, 1
    ux, uy = u % P, u // P
    C[uy + 1, ux + 1] = 0
    sched, rounds = {(ux // TX, uy // TY)}, 0
    for _ in range(max_rounds):
        if not sched:
            break
        assert all(act[b, a] for a, b in sched), "an inactive tile was scheduled"
        rounds += 1
        new_sched, staged = set(), {}
        for (tx, ty) in sorted(sched):
            y0, x0 = ty * TY, tx * TX
            B = C[y0:y0 + TY + 2, x0:x0 + TX + 2].copy()
            M = T[y0 + 1:y0 + TY + 1, x0 + 1:x0 + TX + 1]
            B0 = B[1:-1, 1:-1].copy()
            while True:
                best = B[1:-1, 1:-1].copy()
                for dx, dy in RT.MOVES8:
                    nb = B[1 + dy:TY + 1 + dy, 1 + dx:TX + 1 + dx]
                    np.minimum(best, np.where(nb < big, nb + int(R.chamfer(dx, dy, 0)), big), out=best)
                new = np.where(M, best, B[1:-1, 1:-1])
                if (new == B[1:-1, 1:-1]).all():
                    break
                B[1:-1, 1:-1] = new
            staged[(tx, ty)] = B[1:-1, 1:-1]
            if rounds == 1 or (B[1:-1, 1:-1] != B0).any():
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        a, b = tx + dx, ty + dy
                        if 0 <= a < tp and 0 <= b < tq and act[b, a]:
                            new_sched.add((a, b))
        for (tx, ty), V in staged.items():
            C[ty * TY + 1:ty * TY + TY + 1, tx * TX + 1:tx * TX + TX + 1] = V
        sched = new_sched
    return C[1:Q + 1, 1:P + 1].astype(np.uint32), rounds, int(not sched)


@pytest.mark.parametrize("up", TR.UPS)
def test_converged_matrix_equals_dijkstra_and_is_a_metric(up):
    rng = np.random.default_rng(90 + up)
    shape = [45, 37, 40]
    shape[abs(up) - 1] = 12
    state = scene(rng, shape, up, p_box=0.04, p_hole=0.02)
    origin = (-3, 5, 2)
    terrain = TR.job(state, origin, 0.1, up, 2, 1)
    h0, h1 = RT.plane_axes(up)
    trav = trav_of(terrain)
    Q, P = trav.shape
    cells = rng.choice(np.flatnonzero(trav), size=12, replace=False)
    a = abs(up) - 1
    pts = []
    for c in cells.tolist():
        p = [0.0] * 3
        p[h0], p[h1] = centre(c % P, c // P, 0.1, (origin[h0], origin[h1]))[:2]
        p[a] = float(rng.uniform(-5, 5))
        pts.append(tuple(p))
    info, sites, M = RMT.matrix(terrain, 0.1, pts, 0.0, 1, BIG_TILES)
    assert info["status"] == 0 and (sites["status"] == 0).all() and (sites["converged"] == 1).all()
    assert sites["voxel"].tolist() == cells.tolist() and list(info["origin"]) == list(origin)
    d = dijkstra8(trav, cells)[:, cells]
    assert M.tobytes() == np.where(np.isfinite(d), d, R.INF).astype(np.uint32).tobytes()
    assert (np.diag(M) == 0).all() and (M == M.T).all() and (M != R.INF).any()
    fin = M.astype(np.int64)
    fin[M == R.INF] = 1 << 40
    for k in range(len(cells)):
        assert (fin <= fin[:, k:k + 1] + fin[k:k + 1, :]).all(), k
    exact = RMT.matrix(terrain, 0.1, pts, 0.0, 1, BIG_TILES, exact=True)
    assert exact[2].tobytes() == M.tobytes() and exact[0]["rounds"] == -1


@pytest.mark.parametrize("cap", [1, 7, 40, 4096])
def test_rows_equal_the_terrain_reach_job_from_each_site(cap):
    terrain, fshape = plane(serpentine(48, 100), 0.1, (4, -7, 3))
    trav = trav_of(terrain)
    rng = np.random.default_rng(cap)
    cells = rng.choice(np.flatnonzero(trav), size=6, replace=False).tolist()
    pts = [centre(c % 100, c // 100, 0.1, (4, -7), z=float(rng.uniform(-1, 1))) for c in cells] + [(-5.0, 0.0, 0.0)]
    info, sites, M = RMT.matrix(terrain, 0.1, pts, 0.0, 1, BIG_TILES, max_rounds=cap)
    assert info["status"] == 0 and info["n_active_tiles"] == RMT.active_tiles(trav).sum() == 4 * 3
    assert info["rounds"] == sites["rounds"].max()
    for i, p in enumerate(pts[:-1]):
        rinfo, _, _, cost = RT.job(terrain, fshape, 0.1, p, 0.0, 1, max_rounds=cap)
        assert rinfo["start_voxel"] == sites[i]["voxel"] == cells[i]
        assert (sites[i]["rounds"], sites[i]["converged"], sites[i]["n_reached"]) == \
            (rinfo["rounds"], rinfo["converged"], rinfo["n_reached"])
        assert M[i, :-1].tobytes() == cost.reshape(-1)[cells].tobytes()
    assert cap > 7 or (sites["converged"][:-1] == 0).all()
    assert cap != 4096 or (sites["converged"] == 1).all()
    assert sites[-1]["status"] == 1 and sites[-1]["voxel"] == -1 and (M[-1] == R.INF).all() and (M[:, -1] == R.INF).all()
    assert (sites[-1]["rounds"], sites[-1]["converged"], sites[-1]["n_reached"]) == (0, 1, 0)


def walled(Q, P, p, q):
    """An open plane but for an occupied ring around (p, q), one cell off."""
    st = np.full((Q, P), FREE, np.uint8)
    for dq in range(-2, 3):
        for dp in range(-2, 3):
            if max(abs(dq), abs(dp)) == 2 and 0 <= q + dq < Q and 0 <= p + dp < P:
                st[q + dq, p + dp] = OCCUPIED
    return st


@pytest.mark.parametrize("case", range(6))
def test_active_tile_scheduling_equals_dense_scheduling(case):
    rng = np.random.default_rng(case)
    if case == 0:
        st = rng.choice(np.array([FREE, OCCUPIED, UNKNOWN], np.uint8), size=(37, 75), p=(0.55, 0.3, 0.15))
    elif case == 1:
        st = rng.choice(np.array([FREE, OCCUPIED], np.uint8), size=(1, 130), p=(0.85, 0.15))
    elif case == 2:
        st = rng.choice(np.array([FREE, OCCUPIED], np.uint8), size=(70, 1), p=(0.85, 0.15))
    elif case == 3:
        st = serpentine(48, 100)
    elif case == 4:   # a start walled off in its tile, whose neighbour tiles are partly inactive
        st = np.full((48, 96), OCCUPIED, np.uint8)
        st[16:, :] = FREE
        st[:16, 32:] = FREE
        st[2:5, 2:5] = FREE
        st[0:16, 31] = OCCUPIED
    else:             # walled starts on a tile's corner and edges
        st = walled(40, 70, 31, 15)
    terrain, _ = plane(st)
    trav = trav_of(terrain)
    starts = rng.choice(np.flatnonzero(trav), size=min(3, int(trav.sum())), replace=False).tolist()
    if case == 4:
        starts.append(3 * 96 + 3)
    if case == 5:
        starts.append(15 * 70 + 31)
    for u in starts:
        for rounds in (1, 3, 10, 4096):
            want = RT.emulate(trav, int(u), rounds)
            got = sparse_flat_emulate(trav, int(u), rounds)
            assert got[0].tobytes() == want[0].tobytes() and got[1:] == want[1:], (case, u, rounds)


def test_active_tile_count_by_hand():
    # 75 x 37: flat tiles 3 x 3 (the last column 11 cells wide, the last row 5 high)
    st = np.full((37, 75), OCCUPIED, np.uint8)
    st[0, 0] = FREE      # tile (0, 0)
    st[36, 74] = FREE    # tile (2, 2), the clipped corner
    st[20, 40] = FREE    # tile (1, 1)
    st[31, 63] = FREE    # the same tile again
    st[32, 64] = FREE    # tile (2, 2) again
    act = RMT.active_tiles(trav_of(plane(st)[0]))
    assert act.shape == (3, 3) and act.sum() == 3
    assert act[0, 0] and act[2, 2] and act[1, 1] and not act[0, 1]
    for shape_qp, want in [((1, 1), 1), ((1, 33), 2), ((17, 1), 2), ((16, 32), 1), ((17, 33), 4), ((50, 100), 16)]:
        assert RMT.active_tiles(np.ones(shape_qp, bool)).sum() == want, shape_qp
    # the radius decides: a plane whose clearances fall short of it has no active tile
    st = np.full((5, 6), FREE, np.uint8)
    st[:, ::2] = OCCUPIED
    terrain, _ = plane(st, 0.2)
    assert trav_of(terrain, 0.2).sum() == 15
    info, sites, M = RMT.matrix(terrain, 0.2, [centre(1, 1, 0.2)], 0.6, 4, 1)
    assert info["n_active_tiles"] == 0 and info["n_traversable"] == 0 and info["status"] == 0 and sites[0]["status"] == 2


def test_the_capacity_cut():
    rng = np.random.default_rng(5)
    st = rng.choice(np.array([FREE, OCCUPIED], np.uint8), size=(40, 90), p=(0.7, 0.3))
    terrain, _ = plane(st)
    trav = trav_of(terrain)
    n_active = int(RMT.active_tiles(trav).sum())
    assert n_active == 3 * 3
    pts = [centre(c % 90, c // 90) for c in rng.choice(np.flatnonzero(trav), size=5, replace=False).tolist()]
    ok = RMT.matrix(terrain, 0.1, pts, 0.0, 0, n_active)
    cut = RMT.matrix(terrain, 0.1, pts, 0.0, 0, n_active - 1)
    assert ok[0]["status"] == 0 and (ok[2] != R.INF).any() and ok[0]["rounds"] > 0
    assert cut[0]["status"] == 1 and cut[0]["n_active_tiles"] == n_active and cut[0]["rounds"] == 0
    assert (cut[2] == R.INF).all()
    for f in ("voxel", "status", "approach"):
        assert cut[1][f].tolist() == ok[1][f].tolist(), f
    assert (cut[1]["rounds"] == 0).all() and (cut[1]["converged"] == 0).all() and (cut[1]["n_reached"] == 0).all()


@pytest.mark.parametrize("voxel", [0.05, 0.1, 0.2, 0.3, 0.125, 1.7])
def test_cell_centres_at_any_height_snap_to_themselves(voxel):
    rng = np.random.default_rng(int(voxel * 1000))
    P, Q = 11, 9
    for up in TR.UPS:
        h0, h1 = RT.plane_axes(up)
        a = abs(up) - 1
        for o in [(0, 0, 0), (-5, 7, -3), (1 << 24, -(1 << 24), (1 << 24) - 9), (-(1 << 24) + 3, (1 << 23) + 1, 12345)]:
            for c in rng.integers(0, (P, Q), size=(12, 2)).tolist() + [[0, 0], [P - 1, Q - 1]]:
                p = [0.0] * 3
                p[h0], p[h1] = centre(c[0], c[1], voxel, (o[h0], o[h1]))[:2]
                p[a] = float(rng.choice([-1e7, -3.3, 0.0, 0.04, 1e5]))
                assert R.voxel_of(RT.column_point(p, up, voxel), (o[h0], o[h1], 0), voxel, (P, Q, 1)) == (c[0], c[1], 0), \
                    (voxel, up, o, c)


def test_outside_above_below_blocked_repeated_and_shared_tile_sites():
    P, Q = 40, 20
    st = np.full((Q, P), FREE, np.uint8)
    st[:, 20] = OCCUPIED          # a wall at p = 20 ...
    st[19, 20] = FREE             # ... with a gap at q = 19
    st[5, 30] = OCCUPIED
    terrain, _ = plane(st, 0.5, (2, -3, 7))
    o = (2, -3)
    pts = [centre(1, 1, 0.5, o), centre(2, 1, 0.5, o),              # two sites in one tile
           centre(30, 5, 0.5, o),                                    # a blocked cell: snapped within the window
           centre(1, 1, 0.5, o, z=1e6),                              # a repeat, far above the grid
           centre(1, 1, 0.5, o, z=-1e6),                             # and far below it
           centre(45, 0, 0.5, o),                                    # outside in the plane
           centre(3, -1, 0.5, o, z=3.6),                             # outside in the plane, at the grid's height
           centre(35, 2, 0.5, o)]                                    # beyond the wall
    info, sites, M = RMT.matrix(terrain, 0.5, pts, 0.0, 1, BIG_TILES)
    assert sites["status"].tolist() == [0, 0, 0, 0, 0, 1, 1, 0]
    assert sites[2]["approach"] == 10 and sites[2]["voxel"] != 5 * P + 30
    for k in (3, 4):
        assert M[0].tobytes() == M[k].tobytes() and M[0, k] == 0 and M[k, 0] == 0
    assert M[0, 1] == 10 and (M[5] == R.INF).all() and (M[:, 6] == R.INF).all()
    assert M[0, 7] > 10 * 34   # around the wall through the gap
    info, sites, M = RMT.matrix(terrain, 0.5, pts, 0.0, 0, BIG_TILES)
    assert sites[2]["status"] == 2 and sites[2]["voxel"] == -1 and (M[2] == R.INF).all() and (M[:, 2] == R.INF).all()
    assert (sites[2]["rounds"], sites[2]["converged"], sites[2]["n_reached"]) == (0, 1, 0)


@pytest.mark.parametrize("kw", [dict(radius=float("nan")), dict(radius=-0.1), dict(radius=float("inf")), dict(approach=-1),
                                dict(approach=5), dict(points=[]), dict(points=[(0.0, 0.0, 0.0)] * 3),
                                dict(points=[(0.0, float("nan"), 0.0)]), dict(points=[(float("inf"), 0.0, 0.0)]),
                                dict(points=[(0.0, 0.0, 0.0)] * 2, max_tiles=1 << 15, max_rounds=(1 << 16) + 1)])
def test_refusals(kw):
    terrain, _ = plane(np.full((4, 5), FREE, np.uint8))
    args = dict(points=[(0.0, 0.0, 0.0)], radius=0.0, approach=0, max_tiles=1, max_rounds=1)
    args.update(kw)
    with pytest.raises(ValueError):
        RMT.matrix(terrain, 0.1, args["points"], args["radius"], args["approach"], args["max_tiles"], args["max_rounds"],
                   max_sites=2)
    RMT.matrix(terrain, 0.1, [(0.0, 0.0, 0.0)] * 2, 0.0, 4, 1 << 15, 1 << 16, max_sites=2)   # the work bound itself passes


def test_the_call_is_declared_and_refuses_a_null_context():
    lib = capi.load_library()
    assert "dsm_reach_matrix_enqueue_terrain" in capi.EXPORTS and hasattr(lib, "dsm_reach_matrix_enqueue_terrain")
    pts = np.zeros((1, 3))
    assert lib.dsm_reach_matrix_enqueue_terrain(None, pts.ctypes.data, 1, 0.0, 0) == -1
    assert RMT.SITE_DTYPE == RM.SITE_DTYPE == capi.REACH_SITE_DTYPE
    assert RMT.MATRIX_INFO_DTYPE == RM.MATRIX_INFO_DTYPE == capi.REACH_MATRIX_INFO_DTYPE
