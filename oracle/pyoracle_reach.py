"""The reach job of dsm_reach_enqueue (DESIGN.md §8.11) restated in numpy and scipy: the traversable voxels of a known
field, the start snap, the cost to go (scipy's Dijkstra over the 26-connected chamfer graph, and an emulator of the
device's tile rounds for unconverged jobs), the target records, the paths and the header, in the layout dsm_reach_wait
hands out."""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

UNKNOWN, OCCUPIED, FREE = 0, 1, 2
INF = 0xFFFFFFFF          # UINT32_MAX: not reached
TILE = 8
MAX_CAPACITY = 1 << 26    # DSM_REACH_MAX_CAPACITY
MAX_ROUNDS = 65536        # DSM_REACH_MAX_ROUNDS
MAX_VOXELS = 1 << 27      # DSM_REACH_MAX_VOXELS

TARGET_DTYPE = np.dtype([("cost", "<u4"), ("approach", "<i4"), ("target", "<i4"), ("viewpoint", "<i4"), ("path_offset", "<i4"),
                         ("path_len", "<i4"), ("status", "<i4"), ("reserved", "<i4")])
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("start_voxel", "<i4"), ("start_status", "<i4"), ("start_approach", "<i4"),
                       ("rounds", "<i4"), ("converged", "<i4"), ("n_traversable", "<i4"), ("n_reached", "<i4"),
                       ("n_goals", "<i4"), ("n_clusters_total", "<i4"), ("n_targets", "<i4"), ("n_path_voxels", "<i4"),
                       ("reserved", "<i4", 2)])

# the 26 moves as (dx, dy, dz)
MOVES = [(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy, dz) != (0, 0, 0)]


def chamfer(dx, dy, dz):
    """10 a + 4 b + 3 c for the sorted absolute components a >= b >= c (element-wise on arrays)."""
    d = np.sort(np.abs(np.stack(np.broadcast_arrays(dx, dy, dz)).astype(np.int64)), axis=0)
    return 10 * d[2] + 4 * d[1] + 3 * d[0]


def traversable(state, dist, radius):
    """bool [nz][ny][nx]: free, and the stored fp32 distance >= radius (fp32)."""
    return (np.asarray(state) == FREE) & (np.asarray(dist, np.float32) >= np.float32(radius))


def voxel_of(p, origin, voxel, shape_xyz):
    """floor(p_k / (double)v) - o_k per axis, clamped to [-1, n_k] (outside stays outside)."""
    v = np.float64(np.float32(voxel))
    out = []
    for k in range(3):
        q = np.floor(np.float64(p[k]) / v) - np.float64(origin[k])
        out.append(-1 if q < 0 else shape_xyz[k] if q >= shape_xyz[k] else int(q))
    return tuple(out)


def inside(c, shape_xyz):
    return all(0 <= c[k] < shape_xyz[k] for k in range(3))


def window(c, k, shape_xyz):
    """The window's voxels (x, y, z int arrays) and their offsets from c, clipped to the grid."""
    r = np.arange(-k, k + 1)
    dz, dy, dx = np.meshgrid(r, r, r, indexing="ij")
    x, y, z = c[0] + dx.ravel(), c[1] + dy.ravel(), c[2] + dz.ravel()
    m = (x >= 0) & (x < shape_xyz[0]) & (y >= 0) & (y < shape_xyz[1]) & (z >= 0) & (z < shape_xyz[2])
    return x[m], y[m], z[m], dx.ravel()[m], dy.ravel()[m], dz.ravel()[m]


def snap(trav, s, k):
    """(u, status, approach) of the start voxel s."""
    nz, ny, nx = trav.shape
    if not inside(s, (nx, ny, nz)):
        return -1, 1, 0
    x, y, z, dx, dy, dz = window(s, k, (nx, ny, nz))
    idx = (z * ny + y) * nx + x
    ok = trav.reshape(-1)[idx]
    if not ok.any():
        return -1, 2, 0
    key = chamfer(dx, dy, dz)[ok] * (1 << 32) + idx[ok]
    b = int(key.min())
    return b & 0xFFFFFFFF, 0, b >> 32


def graph(trav):
    """The traversable voxels' 26-connected chamfer graph, a sparse matrix over linear indices (each edge once)."""
    nz, ny, nx = trav.shape
    n = trav.size
    rows, cols, w = [], [], []
    z, y, x = np.nonzero(trav)
    for dx, dy, dz in MOVES:
        if (dz, dy, dx) <= (0, 0, 0):
            continue   # the 13 forward moves
        a, b, c = x + dx, y + dy, z + dz
        m = (a >= 0) & (a < nx) & (b >= 0) & (b < ny) & (c >= 0) & (c < nz)
        m[m] = trav[c[m], b[m], a[m]]
        rows.append((z[m] * ny + y[m]) * nx + x[m])
        cols.append((c[m] * ny + b[m]) * nx + a[m])
        w.append(np.full(int(m.sum()), int(chamfer(dx, dy, dz)), np.float64))
    if not rows:
        return sparse.csr_matrix((n, n))
    return sparse.csr_matrix((np.concatenate(w), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def dijkstra(trav, u):
    """uint32 cost grid of the exact cost to go from linear index u (INF unreached; all INF for u < 0)."""
    cost = np.full(trav.size, INF, np.uint32)
    if u >= 0:
        d = csgraph.dijkstra(graph(trav), directed=False, indices=u)
        f = np.isfinite(d)
        cost[f] = d[f].astype(np.uint32)   # integer sums, exact in fp64
    return cost.reshape(trav.shape)


def emulate(trav, u, max_rounds):
    """(cost, rounds, converged) of the device's tile rounds (include/dsm.h): every scheduled tile relaxes to its
    tile-local fixed point with its halo frozen at the round's start, and a tile that changed (round 0's start tile always
    does) schedules itself and its 26 neighbours.  One grid holds the latest value of every voxel, which is what both device buffers agree on."""
    nz, ny, nx = trav.shape
    tn = [(nx + TILE - 1) // TILE, (ny + TILE - 1) // TILE, (nz + TILE - 1) // TILE]
    P = [tn[2] * TILE + 2, tn[1] * TILE + 2, tn[0] * TILE + 2]
    big = np.int64(INF)
    C = np.full(P, big, np.int64)           # padded by one voxel (and to whole tiles) with INF
    T = np.zeros(P, bool)
    T[1:nz + 1, 1:ny + 1, 1:nx + 1] = trav
    if u < 0:
        return np.full(trav.shape, INF, np.uint32), 0, 1
    ux, uy, uz = u % nx, u // nx % ny, u // (nx * ny)
    C[uz + 1, uy + 1, ux + 1] = 0
    sched = {(ux // TILE, uy // TILE, uz // TILE)}
    rounds = 0
    r = np.arange(TILE + 2)
    for _ in range(max_rounds):
        if not sched:
            break
        rounds += 1
        tiles = np.array(sorted(sched), np.int64)                 # (tx, ty, tz)
        zz = tiles[:, 2, None] * TILE + r[None, :]                # padded coordinates of tile + halo
        yy = tiles[:, 1, None] * TILE + r[None, :]
        xx = tiles[:, 0, None] * TILE + r[None, :]
        B = C[zz[:, :, None, None], yy[:, None, :, None], xx[:, None, None, :]]   # [tiles][10][10][10]
        M = T[zz[:, :, None, None], yy[:, None, :, None], xx[:, None, None, :]][:, 1:-1, 1:-1, 1:-1]
        B0 = B[:, 1:-1, 1:-1, 1:-1].copy()
        while True:
            best = B[:, 1:-1, 1:-1, 1:-1].copy()
            for dx, dy, dz in MOVES:
                nb = B[:, 1 + dz:TILE + 1 + dz, 1 + dy:TILE + 1 + dy, 1 + dx:TILE + 1 + dx]
                np.minimum(best, np.where(nb < big, nb + int(chamfer(dx, dy, dz)), big), out=best)
            new = np.where(M, best, B[:, 1:-1, 1:-1, 1:-1])
            if (new == B[:, 1:-1, 1:-1, 1:-1]).all():
                break
            B[:, 1:-1, 1:-1, 1:-1] = new
        changed = (B[:, 1:-1, 1:-1, 1:-1] != B0).any(axis=(1, 2, 3))
        if rounds == 1:
            changed[:] = True   # the start's seed is round 0's change, whatever the rest of its tile does
        C[zz[:, 1:-1, None, None], yy[:, None, 1:-1, None], xx[:, None, None, 1:-1]] = B[:, 1:-1, 1:-1, 1:-1]
        sched = set()
        for (tx, ty, tz) in tiles[changed].tolist():
            for dz in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        a, b, c = tx + dx, ty + dy, tz + dz
                        if 0 <= a < tn[0] and 0 <= b < tn[1] and 0 <= c < tn[2]:
                            sched.add((a, b, c))
    cost = C[1:nz + 1, 1:ny + 1, 1:nx + 1].astype(np.uint32)
    return cost, rounds, int(not sched)


def best_in_window(trav, cost, g, k):
    """(key, u) of the window of g: the least cost[u] + chamfer(g - u), then u, over reached traversable voxels u; key
    None when there is none."""
    nz, ny, nx = trav.shape
    x, y, z, dx, dy, dz = window(g, k, (nx, ny, nz))
    idx = (z * ny + y) * nx + x
    c = cost.reshape(-1)[idx].astype(np.int64)
    ok = trav.reshape(-1)[idx] & (c != INF)
    if not ok.any():
        return None
    key = (c + chamfer(dx, dy, dz))[ok] * (1 << 32) + idx[ok]
    return int(key.min())


def walk(trav, cost, v):
    """The path start -> v: from v, step to the traversable neighbour p minimising (cost[p] + w(p, x), p)."""
    nz, ny, nx = trav.shape
    flat_t, flat_c = trav.reshape(-1), cost.reshape(-1).astype(np.int64)
    out = [v]
    x = v
    while flat_c[x] != 0:
        px, py, pz = x % nx, x // nx % ny, x // (nx * ny)
        best = None
        for dx, dy, dz in MOVES:
            a, b, c = px + dx, py + dy, pz + dz
            if not (0 <= a < nx and 0 <= b < ny and 0 <= c < nz):
                continue
            p = (c * ny + b) * nx + a
            if not flat_t[p] or flat_c[p] == INF:
                continue
            key = (int(flat_c[p]) + int(chamfer(dx, dy, dz)), p)
            best = key if best is None or key < best else best
        assert best is not None and flat_c[best[1]] < flat_c[x], "the walk's cost must fall"
        x = best[1]
        out.append(x)
    return out[::-1]


def reach(state, dist, origin, voxel, start, radius, approach, goals=(), frontier=None, max_targets=64, max_path=1 << 16,
          max_rounds=MAX_ROUNDS, exact=False):
    """(info INFO_DTYPE record, targets TARGET_DTYPE [n_targets], path int32 [n_path_voxels], cost uint32 [nz][ny][nx])
    of a reach job on the state and distance grids [nz][ny][nx] at integer origin (x, y, z).  frontier: the (clusters,
    voxels) of pyoracle_frontier.frontiers on the same grid, or None.  exact: the cost from Dijkstra, the rounds and
    converged fields are then -1 (the caller checks converged itself); otherwise the tile-round emulator."""
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    shape = (nx, ny, nz)
    trav = traversable(st, dist, radius)
    s = voxel_of(start, origin, voxel, shape)
    u, status, appr = snap(trav, s, approach)
    if exact:
        cost, rounds, conv = dijkstra(trav, u), -1, -1
    else:
        cost, rounds, conv = emulate(trav, u, max_rounds)
    goals = np.asarray(goals, np.float64).reshape(-1, 3)
    ng = len(goals)
    clusters, members = frontier if frontier is not None else (np.zeros(0), np.zeros(0, np.int32))
    n_cl_total = len(clusters)
    n_cl = min(n_cl_total, max_targets - ng)
    recs = np.zeros(ng + n_cl, TARGET_DTYPE)
    recs["cost"], recs["approach"], recs["viewpoint"], recs["path_offset"] = INF, -1, -1, -1
    for t in range(ng):
        g = voxel_of(goals[t], origin, voxel, shape)
        if not inside(g, shape):
            recs[t]["target"], recs[t]["status"] = -1, 1
            continue
        recs[t]["target"] = (g[2] * ny + g[1]) * nx + g[0]
        key = best_in_window(trav, cost, g, approach)
        if key is None:
            recs[t]["status"] = 2
            continue
        recs[t]["cost"], recs[t]["viewpoint"] = key >> 32, key & 0xFFFFFFFF
    for c in range(n_cl):
        t = ng + c
        cl = clusters[c]
        recs[t]["target"] = cl["first"]
        if cl["offset"] < 0:
            recs[t]["status"] = 3
            continue
        best = None
        for gi in members[cl["offset"]:cl["offset"] + cl["n_voxels"]].tolist():   # ascending: ties keep the lowest
            key = best_in_window(trav, cost, (gi % nx, gi // nx % ny, gi // (nx * ny)), approach)
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
        p = walk(trav, cost, int(recs[t]["viewpoint"]))
        recs[t]["path_len"] = len(p)
        if not full and at + len(p) <= max_path:
            recs[t]["path_offset"] = at
            paths += p
            at += len(p)
        else:
            full = True
    info = np.zeros((), INFO_DTYPE)
    info["origin"] = origin
    info["start_voxel"], info["start_status"], info["start_approach"] = u, status, appr
    info["rounds"], info["converged"] = rounds, conv
    info["n_traversable"], info["n_reached"] = int(trav.sum()), int((flat != INF).sum())
    info["n_goals"], info["n_clusters_total"], info["n_targets"], info["n_path_voxels"] = ng, n_cl_total, len(recs), at
    return info, recs, np.asarray(paths, np.int32), cost
