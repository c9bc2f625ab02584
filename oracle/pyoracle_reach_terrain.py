"""The terrain reach job of dsm_reach_enqueue_terrain (DESIGN.md §8.21) restated by composing pyoracle_terrain and
pyoracle_reach: the reach job of §8.11 on the plane (P, Q, 1) of a terrain job's status and clearance planes, with every
point reduced to its column, frontier members standing for their columns' cells, and rounds on flat 32 x 16 tiles
(this module's emulator; the records, paths and header follow pyoracle_reach.reach on the plane's cells)."""
import numpy as np

import pyoracle_reach as R
import pyoracle_terrain as TR
from pyoracle_frontier import CLUSTER_DTYPE as CLUSTER_DTYPE

TX, TY = 32, 16   # the flat tile: cells along p and q
MOVES8 = [(dx, dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy) != (0, 0)]


def plane_axes(up):
    """(h0, h1): the terrain grid's lower and higher in-plane axes."""
    a = abs(up) - 1
    return tuple(k for k in range(3) if k != a)


def check_request(radius, approach, goals, max_targets):
    """Raises ValueError where dsm_reach_enqueue_terrain returns DSM_E_INVALID (exactly dsm_reach_enqueue's checks)."""
    goals = np.asarray(goals, np.float64).reshape(-1, 3)
    if not np.isfinite(radius) or not radius >= 0:
        raise ValueError("radius not finite and >= 0")
    if not 0 <= approach <= 4:
        raise ValueError("approach outside [0, 4]")
    if len(goals) > max_targets:
        raise ValueError("more goals than max_targets")
    if not np.isfinite(goals).all():
        raise ValueError("a goal is not finite")


def column_point(p, up, voxel):
    """A point of the plane grid standing for world point p: its two in-plane coordinates, and the centre of the plane's
    one voxel along the third axis, so that reach's voxel conversion gives (p_h0, p_h1, 0)."""
    h0, h1 = plane_axes(up)
    return (float(p[h0]), float(p[h1]), 0.5 * float(np.float32(voxel)))


def emulate(trav, u, max_rounds):
    """(cost [Q][P], rounds, converged) of the device's rounds on flat tiles of the plane trav [Q][P] (include/dsm.h):
    pyoracle_reach.emulate's rule on 32 x 16 tiles, each relaxing to its tile-local fixed point over the 8 in-plane moves
    with its one-cell halo frozen at the round's start; a tile that changed (round 0's start tile always does) schedules
    itself and its 8 neighbours."""
    Q, P = trav.shape
    tn = [(P + TX - 1) // TX, (Q + TY - 1) // TY]
    big = np.int64(R.INF)
    C = np.full((tn[1] * TY + 2, tn[0] * TX + 2), big, np.int64)   # padded by one cell (and to whole tiles) with INF
    T = np.zeros(C.shape, bool)
    T[1:Q + 1, 1:P + 1] = trav
    if u < 0:
        return np.full(trav.shape, R.INF, np.uint32), 0, 1
    ux, uy = u % P, u // P
    C[uy + 1, ux + 1] = 0
    sched = {(ux // TX, uy // TY)}
    rounds = 0
    rx, ry = np.arange(TX + 2), np.arange(TY + 2)
    for _ in range(max_rounds):
        if not sched:
            break
        rounds += 1
        tiles = np.array(sorted(sched), np.int64)                 # (tx, ty)
        yy = tiles[:, 1, None] * TY + ry[None, :]                 # padded coordinates of tile + halo
        xx = tiles[:, 0, None] * TX + rx[None, :]
        B = C[yy[:, :, None], xx[:, None, :]]                     # [tiles][TY + 2][TX + 2]
        M = T[yy[:, :, None], xx[:, None, :]][:, 1:-1, 1:-1]
        B0 = B[:, 1:-1, 1:-1].copy()
        while True:
            best = B[:, 1:-1, 1:-1].copy()
            for dx, dy in MOVES8:
                nb = B[:, 1 + dy:TY + 1 + dy, 1 + dx:TX + 1 + dx]
                np.minimum(best, np.where(nb < big, nb + int(R.chamfer(dx, dy, 0)), big), out=best)
            new = np.where(M, best, B[:, 1:-1, 1:-1])
            if (new == B[:, 1:-1, 1:-1]).all():
                break
            B[:, 1:-1, 1:-1] = new
        changed = (B[:, 1:-1, 1:-1] != B0).any(axis=(1, 2))
        if rounds == 1:
            changed[:] = True   # the start's seed is round 0's change, whatever the rest of its tile does
        C[yy[:, 1:-1, None], xx[:, None, 1:-1]] = B[:, 1:-1, 1:-1]
        sched = set()
        for (tx, ty) in tiles[changed].tolist():
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    a, b = tx + dx, ty + dy
                    if 0 <= a < tn[0] and 0 <= b < tn[1]:
                        sched.add((a, b))
    return C[1:Q + 1, 1:P + 1].astype(np.uint32), rounds, int(not sched)


def member_cells(voxels, field_shape, up):
    """The cells (q P + p) of the columns of field voxels (linear indices of the field grid (nx, ny, nz))."""
    nx, ny, nz = field_shape
    v = np.asarray(voxels, np.int64)
    c = (v % nx, v // nx % ny, v // (nx * ny))
    h0, h1 = plane_axes(up)
    return (c[h1] * field_shape[h0] + c[h0]).astype(np.int32)


def job(terrain, field_shape, voxel, start, radius, approach, goals=(), frontier=None, max_targets=64, max_path=1 << 16,
        max_rounds=R.MAX_ROUNDS, exact=False):
    """(info, targets, path, cost [m2][m1][m0]) of a terrain reach job, as dsm_reach_wait returns them after
    dsm_reach_enqueue_terrain.  terrain: the (info, level, status, step, clearance) of pyoracle_terrain.job (or of the
    device); field_shape: the field grid (nx, ny, nz) the terrain job read; frontier: the (clusters, voxels) of a frontier
    job on that field, or None.  exact: Dijkstra's costs, rounds and converged -1 (pyoracle_reach.reach)."""
    tinfo, _, status, _, clearance = terrain
    up = int(tinfo["up"])
    m = [int(x) for x in tinfo["m"]]
    h0, h1 = plane_axes(up)
    P, Q = m[h0], m[h1]
    origin = [int(x) for x in tinfo["origin"]]
    plane_origin = (origin[h0], origin[h1], 0)
    st = np.asarray(status, np.uint8).reshape(1, Q, P)
    cl = np.asarray(clearance, np.float32).reshape(1, Q, P)
    goals = np.asarray(goals, np.float64).reshape(-1, 3)
    check_request(radius, approach, goals, max_targets)
    fr = None
    if frontier is not None:
        clusters, members = frontier
        clusters = np.array(clusters, copy=True)
        if len(clusters):
            clusters["first"] = member_cells(clusters["first"], field_shape, up)
        fr = (clusters, member_cells(members, field_shape, up))
    shape = (P, Q, 1)
    trav = R.traversable(st, cl, radius)
    u, start_status, appr = R.snap(trav, R.voxel_of(column_point(start, up, voxel), plane_origin, voxel, shape), approach)
    if exact:
        cost, rounds, conv = R.dijkstra(trav, u), -1, -1
    else:
        cost, rounds, conv = emulate(trav[0], u, max_rounds)
    cost = cost.reshape(1, Q, P)
    # the targets, records, paths and header: pyoracle_reach.reach's, on the plane's cells
    ng = len(goals)
    clusters, cmembers = fr if fr is not None else (np.zeros(0, CLUSTER_DTYPE), np.zeros(0, np.int32))
    n_clustertotal = len(clusters)
    n_cl = min(n_clustertotal, max_targets - ng)
    recs = np.zeros(ng + n_cl, R.TARGET_DTYPE)
    recs["cost"], recs["approach"], recs["viewpoint"], recs["path_offset"] = R.INF, -1, -1, -1
    for t in range(ng):
        g = R.voxel_of(column_point(goals[t], up, voxel), plane_origin, voxel, shape)
        if not R.inside(g, shape):
            recs[t]["target"], recs[t]["status"] = -1, 1
            continue
        recs[t]["target"] = g[1] * P + g[0]
        key = R.best_in_window(trav, cost, g, approach)
        if key is None:
            recs[t]["status"] = 2
            continue
        recs[t]["cost"], recs[t]["viewpoint"] = key >> 32, key & 0xFFFFFFFF
    for c in range(n_cl):
        t = ng + c
        cluster = clusters[c]
        recs[t]["target"] = cluster["first"]
        if cluster["offset"] < 0:
            recs[t]["status"] = 3
            continue
        best = None
        for gi in cmembers[cluster["offset"]:cluster["offset"] + cluster["n_voxels"]].tolist():   # field order: ties keep the lowest
            key = R.best_in_window(trav, cost, (gi % P, gi // P, 0), approach)
            if key is not None and (best is None or key < best[0]):
                best = (key, gi)
        if best is None:
            recs[t]["status"] = 2
            continue
        recs[t]["cost"], recs[t]["viewpoint"], recs[t]["target"] = best[0] >> 32, best[0] & 0xFFFFFFFF, best[1]
    flat = cost.reshape(-1)
    ok = recs["status"] == 0
    recs["approach"][ok] = recs["cost"][ok].astype(np.int64) - flat[recs["viewpoint"][ok]].astype(np.int64)
    paths, at, full = [], 0, False
    for t in range(len(recs)):
        if recs[t]["status"] != 0:
            continue
        pth = R.walk(trav, cost, int(recs[t]["viewpoint"]))
        recs[t]["path_len"] = len(pth)
        if not full and at + len(pth) <= max_path:
            recs[t]["path_offset"] = at
            paths += pth
            at += len(pth)
        else:
            full = True
    info = np.zeros((), R.INFO_DTYPE)
    info["origin"] = origin
    info["start_voxel"], info["start_status"], info["start_approach"] = u, start_status, appr
    info["rounds"], info["converged"] = rounds, conv
    info["n_traversable"], info["n_reached"] = int(trav.sum()), int((flat != R.INF).sum())
    info["n_goals"], info["n_clusters_total"], info["n_targets"], info["n_path_voxels"] = ng, n_clustertotal, len(recs), at
    return info, recs, np.asarray(paths, np.int32), cost.reshape(m[2], m[1], m[0])


def from_state(state, origin, voxel, up, headroom, max_step, *args, **kw):
    """A terrain job on the state grid [nz][ny][nx] (pyoracle_terrain.job), then the terrain reach job on it: (terrain,
    reach) with reach the tuple of job()."""
    terrain = TR.job(state, origin, voxel, up, headroom, max_step)
    nz, ny, nx = np.asarray(state).shape
    return terrain, job(terrain, (nx, ny, nz), voxel, *args, **kw)
