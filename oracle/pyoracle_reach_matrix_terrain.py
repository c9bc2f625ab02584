"""The terrain matrix job of dsm_reach_matrix_enqueue_terrain (DESIGN.md §8.22) composed from its parts: every site
reduced to its column (pyoracle_reach_terrain.column_point) and snapped on the plane (pyoracle_reach.snap), each row the
flat-tile round emulator started at that site (pyoracle_reach_terrain.emulate), the active 32 x 16 tiles and the
capacity cut, in the dtypes and layout of pyoracle_reach_matrix, as dsm_reach_matrix_wait hands them out."""
import numpy as np
from scipy.sparse import csgraph

import pyoracle_reach as R
import pyoracle_reach_terrain as RT
from pyoracle_reach_matrix import MATRIX_INFO_DTYPE, MAX_SITES, SITE_DTYPE

MAX_WORK = 1 << 32   # DSM_REACH_MATRIX_MAX_WORK


def active_tiles(trav):
    """The flat tiles (32 x 16 cells from cell (0, 0), edge tiles clipped) of the plane trav [Q][P] holding a traversable
    cell: bool [tq][tp]."""
    Q, P = trav.shape
    pad = np.zeros(((Q + RT.TY - 1) // RT.TY * RT.TY, (P + RT.TX - 1) // RT.TX * RT.TX), bool)
    pad[:Q, :P] = trav
    return pad.reshape(pad.shape[0] // RT.TY, RT.TY, pad.shape[1] // RT.TX, RT.TX).any(axis=(1, 3))


def check_request(points, radius, approach, max_sites, max_tiles, max_rounds):
    """Raises ValueError where dsm_reach_matrix_enqueue_terrain returns DSM_E_INVALID (exactly dsm_reach_matrix_enqueue's
    checks)."""
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    if not np.isfinite(radius) or not radius >= 0:
        raise ValueError("radius not finite and >= 0")
    if not 0 <= approach <= 4:
        raise ValueError("approach outside [0, 4]")
    if not 1 <= len(pts) <= max_sites:
        raise ValueError("n_points outside [1, max_sites]")
    if len(pts) * max_tiles * max_rounds > MAX_WORK:
        raise ValueError("n_points x max_tiles x max_rounds above 2^32")
    if not np.isfinite(pts).all():
        raise ValueError("a point is not finite")


def plane(terrain, radius):
    """(trav [Q][P], up, (P, Q), the plane's origin (o_h0, o_h1, 0)) of a terrain job's result at `radius`."""
    tinfo, _, status, _, clearance = terrain
    up = int(tinfo["up"])
    h0, h1 = RT.plane_axes(up)
    P, Q = int(tinfo["m"][h0]), int(tinfo["m"][h1])
    st = np.asarray(status, np.uint8).reshape(1, Q, P)
    cl = np.asarray(clearance, np.float32).reshape(1, Q, P)
    return R.traversable(st, cl, radius)[0], up, (P, Q), (int(tinfo["origin"][h0]), int(tinfo["origin"][h1]), 0)


def snap(terrain, voxel, points, radius, approach):
    """The sites' (cell, status, approach) as a terrain reach job snaps its start."""
    trav, up, (P, Q), o = plane(terrain, radius)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    return [R.snap(trav[None], R.voxel_of(RT.column_point(p, up, voxel), o, voxel, (P, Q, 1)), approach) for p in pts]


def matrix(terrain, voxel, points, radius, approach, max_tiles, max_rounds=R.MAX_ROUNDS, max_sites=MAX_SITES, exact=False):
    """(info MATRIX_INFO_DTYPE record, sites SITE_DTYPE [n], M uint32 [n][n]) of a terrain matrix job on terrain, the
    (info, level, status, step, clearance) of pyoracle_terrain.job (or of the device), with voxel edge `voxel`: row i is
    the terrain reach job from site i (pyoracle_reach_terrain.emulate) read at the sites.  The cut: more active flat tiles
    than max_tiles.  exact: Dijkstra's rows, with rounds and converged -1 in the records and the header."""
    check_request(points, radius, approach, max_sites, max_tiles, max_rounds)
    trav, _, (P, Q), _ = plane(terrain, radius)
    snaps = snap(terrain, voxel, points, radius, approach)
    n = len(snaps)
    n_active = int(active_tiles(trav).sum())
    cut = n_active > max_tiles
    sites = np.zeros(n, SITE_DTYPE)
    M = np.full((n, n), R.INF, np.uint32)
    rounds = 0
    us = [u for u, _, _ in snaps]
    if exact and not cut:
        rows = {}
        starts = sorted({u for u in us if u >= 0})
        if starts:
            d = csgraph.dijkstra(R.graph(trav[None]), directed=False, indices=starts)
            for k, u in enumerate(starts):
                c = np.full(trav.size, R.INF, np.uint32)
                f = np.isfinite(d[k])
                c[f] = d[k][f].astype(np.uint32)
                rows[u] = c
    for i, (u, status, appr) in enumerate(snaps):
        sites[i]["voxel"], sites[i]["status"], sites[i]["approach"] = u, status, appr
        if cut:
            continue
        if exact:
            flat = rows[u] if u >= 0 else np.full(trav.size, R.INF, np.uint32)
            r, conv = (-1, -1) if u >= 0 else (0, 1)
        else:
            cost, r, conv = RT.emulate(trav, u, max_rounds)
            flat = cost.reshape(-1)
        sites[i]["rounds"], sites[i]["converged"], sites[i]["n_reached"] = r, conv, int((flat != R.INF).sum())
        rounds = max(rounds, r)
        if u >= 0:
            for j, v in enumerate(us):
                if v >= 0:
                    M[i, j] = flat[v]
    info = np.zeros((), MATRIX_INFO_DTYPE)
    info["origin"] = terrain[0]["origin"]
    info["n_sites"], info["status"] = n, int(cut)
    info["n_traversable"], info["n_active_tiles"], info["max_tiles"] = int(trav.sum()), n_active, max_tiles
    info["rounds"] = -1 if exact and not cut else rounds
    return info, sites, M
