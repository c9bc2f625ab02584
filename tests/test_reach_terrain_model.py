"""The terrain reach model of oracle/pyoracle_reach_terrain (DESIGN.md §8.21) on the CPU: converged jobs against scipy's
Dijkstra on the 8-connected 10/14 graph for all six up axes and against the 8x8x8 rounds of §8.11, the flat tile's round
counts counted by hand, walled-off starts on tile edges and corners, unconverged bounds, points above, below and
beside the grid, frontier members sharing a column and their ties, both capacity cuts, and every refusal."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

import pyoracle_field_known
import pyoracle_frontier
import pyoracle_reach as R
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR

FREE, OCCUPIED, UNKNOWN = R.FREE, R.OCCUPIED, R.UNKNOWN


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
    pos = {h1: 0, h0: 1, a: 2}                                  # grid axis -> axis of col ([h1][h0][a])
    return np.ascontiguousarray(np.transpose(col, (pos[2], pos[1], pos[0])))


def plane(status, voxel=0.1, origin=(0, 0, 0), n_up=4):
    """A terrain job's result (up = +3) with the given status plane [Q][P]: the terrain grid (P, Q, 1) of a field
    (P, Q, n_up); the clearance is the known field's distance of the status plane, as the terrain job computes it."""
    st = np.asarray(status, np.uint8)[None]
    clear, n_blocked, n_trav = pyoracle_field_known.state_field(st, voxel)
    info = np.zeros(1, TR.INFO_DTYPE)[0]
    info["origin"], info["m"], info["up"] = origin, (st.shape[2], st.shape[1], 1), 3
    return (info, None, st, None, clear), (st.shape[2], st.shape[1], n_up)


def centre(p, q, voxel=0.1, origin=(0, 0, 0), z=0.0):
    return ((p + origin[0] + 0.5) * float(np.float32(voxel)), (q + origin[1] + 0.5) * float(np.float32(voxel)), z)


def dijkstra8(trav, u):
    """uint32 [Q][P]: the exact cost to go over the 8-connected 10/14 graph of trav [Q][P], an independent restatement."""
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
    d = csgraph.dijkstra(g, directed=False, indices=u)
    out = np.full(trav.size, R.INF, np.uint32)
    f = np.isfinite(d)
    out[f] = d[f].astype(np.uint32)
    return out.reshape(trav.shape)


def plane_shape(info):
    up = int(info["up"])
    h0, h1 = RT.plane_axes(up)
    return int(info["m"][h1]), int(info["m"][h0])


@pytest.mark.parametrize("up", TR.UPS)
def test_converged_jobs_are_dijkstra_on_the_8_connected_graph(up):
    rng = np.random.default_rng(70 + up)
    shape = [45, 37, 40]
    shape[abs(up) - 1] = 12
    state = scene(rng, shape, up, p_box=0.03, p_hole=0.02)
    for radius in (0.0, 0.1):
        start = [(shape[k] // 2 + 0.5) * 0.1 for k in range(3)]
        goals = [[(rng.integers(0, shape[k]) + 0.5) * 0.1 for k in range(3)] for _ in range(6)]
        terrain, (info, recs, path, cost) = RT.from_state(state, (0, 0, 0), 0.1, up, 2, 1, start, radius, 1, goals)
        assert info["converged"] == 1
        Q, P = plane_shape(terrain[0])
        trav = R.traversable(terrain[2], terrain[4], radius).reshape(Q, P)
        assert trav.sum() > 0.3 * trav.size
        u = int(info["start_voxel"])
        assert u >= 0 and info["start_status"] == 0
        assert (cost.reshape(Q, P) == dijkstra8(trav, u)).all()
        assert int(info["n_reached"]) == int((cost != R.INF).sum()) and (recs["status"] == 0).any()
        for r in recs[recs["status"] == 0]:
            seg = path[r["path_offset"]:r["path_offset"] + r["path_len"]]
            assert seg[0] == u and seg[-1] == r["viewpoint"]
            assert trav[seg // P, seg % P].all()
            steps = np.abs(np.diff(seg // P)) + np.abs(np.diff(seg % P))
            weight = sum(10 if s == 1 else 14 for s in steps)
            assert weight == cost.reshape(-1)[r["viewpoint"]]


def test_converged_flat_tiles_equal_the_field_jobs_tiles():
    """On converged grids the terrain job is pyoracle_reach on the status and clearance planes as a one-voxel-thick
    known field, rounds on 8x8x8 tiles or flat ones alike; only the round count differs."""
    rng = np.random.default_rng(5)
    st = rng.choice(np.array([FREE, OCCUPIED, UNKNOWN], np.uint8), size=(70, 90), p=(0.8, 0.12, 0.08))
    terrain, fshape = plane(st, 0.1, (-4, 6, 2))
    start = centre(3, 4, 0.1, (-4, 6, 2))
    goals = [centre(80, 60, 0.1, (-4, 6, 2)), centre(10, 69, 0.1, (-4, 6, 2), z=-50.0)]
    got = RT.job(terrain, fshape, 0.1, start, 0.0, 2, goals)
    field = R.reach(terrain[2], terrain[4], (-4, 6, 0), 0.1, RT.column_point(start, 3, 0.1), 0.0, 2,
                    [RT.column_point(g, 3, 0.1) for g in goals])
    assert got[0]["converged"] == 1 and field[0]["converged"] == 1 and got[0]["rounds"] < field[0]["rounds"]
    for k, (g, w) in enumerate(zip(got, field)):
        g, w = np.array(g, copy=True), np.array(w, copy=True)
        if k == 0:
            g["rounds"] = w["rounds"]
            w["origin"] = g["origin"]
            assert list(g["origin"]) == [-4, 6, 2]
        assert g.tobytes() == w.reshape(g.shape).tobytes(), k


@pytest.mark.parametrize("P,Q,flat,field", [(100, 1, 5, 14), (1, 50, 5, 8), (64, 1, 3, 9), (33, 17, 3, 6)])
def test_flat_tile_round_counts_counted_by_hand(P, Q, flat, field):
    """A start at cell (0, 0) of an open plane: the front crosses one tile per round, and one more round finds no change.
    A row of 100 cells crosses 4 tiles of 32 (13 of 8), a column of 50 crosses 4 of 16 (7 of 8); a 33 x 17 plane needs
    the diagonal tile (1, 1) at round 2."""
    terrain, fshape = plane(np.full((Q, P), FREE, np.uint8))
    info = RT.job(terrain, fshape, 0.1, centre(0, 0), 0.0, 0)[0]
    assert (info["rounds"], info["converged"]) == (flat, 1)
    cost, rounds, conv = R.emulate(np.ones((1, Q, P), bool), 0, 1000)
    assert (rounds, conv) == (field, 1)
    for cap in range(1, flat):
        assert RT.job(terrain, fshape, 0.1, centre(0, 0), 0.0, 0, max_rounds=cap)[0]["converged"] == 0


@pytest.mark.parametrize("p,q", [(5, 5), (31, 7), (32, 7), (31, 15), (32, 16), (0, 0)])
def test_walled_starts_on_tile_edges_and_corners(p, q):
    """A start walled off inside its tile except one gap, on a tile edge, on a corner, and shut in completely."""
    st = np.full((40, 70), FREE, np.uint8)
    ring = [(q + dq, p + dp) for dq in (-2, -1, 0, 1, 2) for dp in (-2, -1, 0, 1, 2) if max(abs(dq), abs(dp)) == 2]
    for a, b in ring:
        if 0 <= a < 40 and 0 <= b < 70:
            st[a, b] = OCCUPIED
    gap = ring[-1]
    terrain, fshape = plane(st)
    for closed in (False, True):
        s = st.copy()
        if not closed:
            s[gap] = FREE
        terrain, fshape = plane(s)
        info, recs, path, cost = RT.job(terrain, fshape, 0.1, centre(p, q), 0.0, 0, [centre(69, 39)])
        trav = R.traversable(terrain[2], terrain[4], 0.0)[0]
        assert info["converged"] == 1
        assert (cost[0] == dijkstra8(trav, q * 70 + p)).all()
        inside = sum(1 for dq in (-1, 0, 1) for dp in (-1, 0, 1) if 0 <= q + dq < 40 and 0 <= p + dp < 70)
        if closed and all(0 <= a < 40 and 0 <= b < 70 for a, b in ring):
            # round 1 reaches the enclosure in the start's tile; a tile holding the rest of it changes in round 2
            one_tile = (p - 1) // 32 == (p + 1) // 32 and (q - 1) // 16 == (q + 1) // 16
            assert info["n_reached"] == inside and recs[0]["status"] == 2 and info["rounds"] == (2 if one_tile else 3)
        if not closed and gap[0] < 40 and gap[1] < 70 and min(gap) >= 0:
            assert recs[0]["status"] == 0


def test_unconverged_results_bound_the_exact_costs():
    """Cut short, a serpentine plane's costs are upper bounds, each reached path's weight lies between the exact cost and
    the reported one, and the paths still step between traversable 8-neighbours down to the start."""
    Q, P = 48, 100
    st = np.full((Q, P), FREE, np.uint8)
    for i, q in enumerate(range(3, Q - 1, 4)):
        st[q, :] = OCCUPIED
        st[q, (P - 1 if i % 2 == 0 else 0)] = FREE
    terrain, fshape = plane(st)
    trav = R.traversable(terrain[2], terrain[4], 0.0)[0]
    exact = dijkstra8(trav, 0).reshape(-1).astype(np.int64)
    goals = [centre(p, q) for q in range(0, Q, 7) for p in range(0, P, 13)]
    seen = 0
    for cap in (2, 5, 9, 30):
        info, recs, path, cost = RT.job(terrain, fshape, 0.1, centre(0, 0), 0.0, 0, goals, max_rounds=cap)
        assert info["converged"] == 0 and info["rounds"] == cap
        c = cost.reshape(-1).astype(np.int64)
        assert (c >= exact).all()
        for r in recs[recs["status"] == 0]:
            seg = path[r["path_offset"]:r["path_offset"] + r["path_len"]]
            steps = np.maximum(np.abs(np.diff(seg // P)), np.abs(np.diff(seg % P)))
            assert (steps == 1).all() and trav.reshape(-1)[seg].all() and seg[0] == 0
            diag = (np.abs(np.diff(seg // P)) + np.abs(np.diff(seg % P))) == 2
            weight = int(10 * (~diag).sum() + 14 * diag.sum())
            assert exact[r["viewpoint"]] <= weight <= c[r["viewpoint"]]
            seen += 1
    assert seen > 10


@pytest.mark.parametrize("up", (-2, 3, 1))
def test_points_stand_for_their_columns(up):
    """A start or goal above or below the grid along up is still in its column; a point outside in the plane has
    status 1 whatever its height."""
    rng = np.random.default_rng(9)
    shape = [30, 26, 22]
    shape[abs(up) - 1] = 10
    state = scene(rng, shape, up, p_box=0.0, p_hole=0.0)
    a = abs(up) - 1
    origin = (3, -4, 5)
    base = [(shape[k] // 2 + origin[k] + 0.5) * 0.1 for k in range(3)]
    goal = [(2 + origin[k] + 0.5) * 0.1 for k in range(3)]
    ref = RT.from_state(state, origin, 0.1, up, 2, 1, base, 0.0, 0, [goal])[1]
    assert ref[0]["start_status"] == 0 and ref[1][0]["status"] == 0
    for h in (-1000.0, -0.05, 1e6):
        s, g = list(base), list(goal)
        s[a], g[a] = h, -h
        got = RT.from_state(state, origin, 0.1, up, 2, 1, s, 0.0, 0, [g])[1]
        for x, y in zip(got, ref):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    h0, _ = RT.plane_axes(up)
    s, g = list(base), list(goal)
    s[h0] = g[h0] = -100.0
    info, recs, _, cost = RT.from_state(state, origin, 0.1, up, 2, 1, s, 0.0, 0, [g, base])[1]
    assert (info["start_status"], info["start_voxel"], info["n_reached"]) == (1, -1, 0)
    assert (recs["status"][0], recs["target"][0]) == (1, -1) and recs["status"][1] == 2
    assert (cost == R.INF).all()


def frontier(members_xyz, field_shape, sizes):
    """A frontier job's (clusters, voxels) for clusters of the given member voxels (x, y, z), listed ascending per
    cluster; a size of 0 is a cluster without listed members."""
    nx, ny, _ = field_shape
    tab = np.zeros(len(sizes), pyoracle_frontier.CLUSTER_DTYPE)
    voxels, at = [], 0
    for c, n in enumerate(sizes):
        idx = sorted((z * ny + y) * nx + x for x, y, z in members_xyz[at:at + max(n, 1)])
        tab[c]["first"] = idx[0]
        tab[c]["n_voxels"] = len(idx)
        tab[c]["offset"] = len(voxels) if n > 0 else -1
        if n > 0:
            voxels += idx
        at += max(n, 1)
    return tab, np.asarray(voxels, np.int32)


def test_frontier_members_share_columns_and_tie_in_the_fields_order():
    """Two members of one cluster tie on (cost, viewpoint) from different columns: the lower member in the field's voxel
    order wins although its cell is the higher one.  Members sharing a column, a cluster without members (status 3,
    target the cell of its first voxel) and one out of reach (status 2)."""
    P, Q = 20, 20
    st = np.full((Q, P), FREE, np.uint8)
    st[:, 10:13] = OCCUPIED
    for q in (8, 9, 11, 12):
        st[q, 9] = OCCUPIED
    st[:, 17] = OCCUPIED      # the strip x 18..19 is cut off
    terrain, fshape = plane(st, n_up=6)
    members = [(10, 11, 1), (10, 9, 5),              # the tie: (10, 11) lower in the field's order
               (4, 4, 0), (4, 4, 3), (4, 4, 5),      # one column, three heights
               (7, 7, 2),                            # a cluster without listed members
               (19, 3, 0), (19, 5, 4)]               # out of reach
    fr = frontier(members, fshape, [2, 3, 0, 2])
    info, recs, path, cost = RT.job(terrain, fshape, 0.1, centre(0, 10), 0.0, 1, frontier=fr)
    assert info["n_targets"] == 4 and info["n_clusters_total"] == 4
    assert recs[0]["status"] == 0 and recs[0]["viewpoint"] == 10 * P + 9 and recs[0]["target"] == 11 * P + 10
    assert recs[0]["cost"] == cost.reshape(-1)[10 * P + 9] + 14 and recs[0]["approach"] == 14
    assert recs[1]["status"] == 0 and recs[1]["target"] == 4 * P + 4 and recs[1]["approach"] == 0
    assert (recs[2]["status"], recs[2]["target"]) == (3, 7 * P + 7)
    assert (recs[3]["status"], recs[3]["target"]) == (2, 3 * P + 19)
    # the same job with the tie's heights swapped picks the other column
    members[0], members[1] = (10, 11, 5), (10, 9, 1)
    recs2 = RT.job(terrain, fshape, 0.1, centre(0, 10), 0.0, 1, frontier=frontier(members, fshape, [2, 3, 0, 2]))[1]
    assert recs2[0]["target"] == 9 * P + 10 and recs2[0]["cost"] == recs[0]["cost"]


def test_capacity_cuts():
    """max_targets drops the clusters past it (n_clusters_total keeps them all); max_path lists a prefix of the paths."""
    st = np.full((30, 40), FREE, np.uint8)
    terrain, fshape = plane(st, n_up=3)
    members = [(5 + 4 * i, 20, 0) for i in range(6)]
    fr = frontier(members, fshape, [1] * 6)
    goals = [centre(39, 29), centre(20, 0)]
    info, recs, path, _ = RT.job(terrain, fshape, 0.1, centre(0, 0), 0.0, 0, goals, fr, max_targets=5, max_path=60)
    assert (info["n_targets"], info["n_goals"], info["n_clusters_total"]) == (5, 2, 6)
    assert (recs["status"] == 0).all()
    lens = recs["path_len"]
    assert recs["path_offset"][0] == 0 and lens[0] == 40 and lens[1] == 21   # 39 diagonal steps and 29 straight; 20 straight
    listed = recs["path_offset"] >= 0
    assert listed[0] and not listed.all() and (np.flatnonzero(~listed).min() > np.flatnonzero(listed).max())
    assert info["n_path_voxels"] == lens[listed].sum() <= 60 and len(path) == info["n_path_voxels"]


@pytest.mark.parametrize("kw", [dict(radius=float("nan")), dict(radius=-0.1), dict(radius=float("inf")), dict(approach=-1),
                                dict(approach=5), dict(goals=[(0.0, 0.0, 0.0)] * 3), dict(goals=[(0.0, float("nan"), 0.0)]),
                                dict(goals=[(float("inf"), 0.0, 0.0)])])
def test_refusals(kw):
    terrain, fshape = plane(np.full((4, 5), FREE, np.uint8))
    args = dict(radius=0.0, approach=0, goals=())
    args.update(kw)
    with pytest.raises(ValueError):
        RT.job(terrain, fshape, 0.1, centre(0, 0), args["radius"], args["approach"], args["goals"], max_targets=2)
    RT.job(terrain, fshape, 0.1, centre(0, 0), 0.0, 4, [(0.0, 0.0, 0.0)] * 2, max_targets=2)
