"""The matrix job of dsm_reach_matrix_enqueue (DESIGN.md §8.13) on top of oracle/pyoracle_reach: the sites snapped as a
reach job's start (pyoracle_reach.snap), each row the round emulator started at that site (pyoracle_reach.emulate), the
active-tile count and the capacity cut, in the layout dsm_reach_matrix_wait hands out."""
import numpy as np

from pyoracle_reach import INF, MAX_ROUNDS, TILE, emulate, snap, traversable, voxel_of

MAX_SITES = 1024          # DSM_REACH_MATRIX_MAX_SITES
SITE_DTYPE = np.dtype([("voxel", "<i4"), ("status", "<i4"), ("approach", "<i4"), ("rounds", "<i4"), ("converged", "<i4"),
                       ("n_reached", "<i4"), ("reserved", "<i4", 2)])
MATRIX_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_sites", "<i4"), ("status", "<i4"), ("n_traversable", "<i4"),
                              ("n_active_tiles", "<i4"), ("max_tiles", "<i4"), ("rounds", "<i4"), ("reserved", "<i4", 7)])


def active_tiles(trav):
    """The tiles (8x8x8 from voxel 0, edge tiles clipped) holding a traversable voxel: bool [tz][ty][tx]."""
    nz, ny, nx = trav.shape
    pad = np.zeros(((nz + TILE - 1) // TILE * TILE, (ny + TILE - 1) // TILE * TILE, (nx + TILE - 1) // TILE * TILE), bool)
    pad[:nz, :ny, :nx] = trav
    tz, ty, tx = (s // TILE for s in pad.shape)
    return pad.reshape(tz, TILE, ty, TILE, tx, TILE).any(axis=(1, 3, 5))


def matrix(state, dist, origin, voxel, points, radius, approach, max_tiles, max_rounds=MAX_ROUNDS):
    """(info MATRIX_INFO_DTYPE record, sites SITE_DTYPE [n], M uint32 [n][n]) of a matrix job on the state and distance
    grids [nz][ny][nx] at integer origin (x, y, z): each site is snapped as a reach job's start, and row i is the
    emulated reach job from site i, read at the sites.  The cut: more active tiles than max_tiles."""
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    trav = traversable(st, dist, radius)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(pts)
    n_active = int(active_tiles(trav).sum())
    cut = n_active > max_tiles
    sites = np.zeros(n, SITE_DTYPE)
    M = np.full((n, n), INF, np.uint32)
    rounds = 0
    snaps = [snap(trav, voxel_of(p, origin, voxel, (nx, ny, nz)), approach) for p in pts]
    for i, (u, status, appr) in enumerate(snaps):
        sites[i]["voxel"], sites[i]["status"], sites[i]["approach"] = u, status, appr
        if cut:
            continue
        cost, r, conv = emulate(trav, u, max_rounds)
        flat = cost.reshape(-1)
        sites[i]["rounds"], sites[i]["converged"], sites[i]["n_reached"] = r, conv, int((flat != INF).sum())
        rounds = max(rounds, r)
        if u >= 0:
            for j, (v, _, _) in enumerate(snaps):
                if v >= 0:
                    M[i, j] = flat[v]
    info = np.zeros((), MATRIX_INFO_DTYPE)
    info["origin"] = origin
    info["n_sites"], info["status"] = n, int(cut)
    info["n_traversable"], info["n_active_tiles"], info["max_tiles"] = int(trav.sum()), n_active, max_tiles
    info["rounds"] = rounds
    return info, sites, M
