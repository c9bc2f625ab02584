"""The viewpoint job of dsm_viewpoint_enqueue (DESIGN.md §8.15) restated in numpy: per frontier cluster, the clear
candidate positions around its centre voxel, each scored at its best rotation by the sampled members it would see
through gain's frustum test and walk (pyoracle_gain.frustum and pyoracle_gain.seen), and the best top_k of them, with
the header and the records in the layout dsm_viewpoint_wait hands out."""
from collections import namedtuple

import numpy as np

import pyoracle_gain as G
import pyoracle_reach

INF = 0xFFFFFFFF
MAX_CLUSTERS = 4096          # DSM_VIEWPOINT_MAX_CLUSTERS
MAX_CANDIDATES = 1 << 22     # DSM_VIEWPOINT_MAX_CANDIDATES
MAX_OFFSETS = 4096           # DSM_VIEWPOINT_MAX_OFFSETS
MAX_ROTATIONS = 64           # DSM_VIEWPOINT_MAX_ROTATIONS
MAX_RADIUS = 64              # DSM_VIEWPOINT_MAX_RADIUS
MAX_DZ = 16                  # DSM_VIEWPOINT_MAX_DZ
MAX_STRIDE = 8               # DSM_VIEWPOINT_MAX_STRIDE
MAX_SAMPLES = 4096           # DSM_VIEWPOINT_MAX_SAMPLES
MAX_TOP_K = 16               # DSM_VIEWPOINT_MAX_TOP_K
MAX_WORK = 1 << 31           # DSM_VIEWPOINT_MAX_WORK

CLUSTER_DTYPE = np.dtype([("cluster", "<i4"), ("status", "<i4"), ("n_samples", "<i4"), ("n_inside", "<i4"), ("n_traversable", "<i4"),
                          ("n_reached", "<i4"), ("n_viewpoints", "<i4"), ("reserved", "<i4")])
VIEWPOINT_DTYPE = np.dtype([("voxel", "<i4"), ("offset", "<i4"), ("rotation", "<i4"), ("n_seen", "<i4"), ("cost", "<u4"),
                            ("reserved", "<i4", 3)])
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_clusters", "<i4"), ("n_offsets", "<i4"), ("n_rotations", "<i4"), ("top_k", "<i4"),
                       ("unknown_blocks", "<i4"), ("with_reach", "<i4"), ("n_clusters_table", "<i4"), ("reserved", "<i4", 6)])

Params = namedtuple("Params", "r_min r_max dz_max stride max_samples min_seen top_k with_reach radius")


def offsets(p):
    """int64 (n, 3): the offsets (dx, dy, dz) in their order, dz outermost, then dy, then dx, each ascending."""
    p = Params(*p)
    s = p.stride
    out = [(dx, dy, dz) for dz in range(-(p.dz_max // s) * s, p.dz_max + 1, s)
           for dy in range(-(p.r_max // s) * s, p.r_max + 1, s)
           for dx in range(-(p.r_max // s) * s, p.r_max + 1, s)
           if p.r_min * p.r_min <= dx * dx + dy * dy <= p.r_max * p.r_max]
    return np.array(out, np.int64).reshape(-1, 3)


def check_enable(max_clusters, max_candidates):
    """Raises ValueError where dsm_viewpoint_enable returns DSM_E_INVALID."""
    if not (1 <= max_clusters <= MAX_CLUSTERS and 1 <= max_candidates <= MAX_CANDIDATES):
        raise ValueError("max_clusters outside [1, 4096] or max_candidates outside [1, 2^22]")


def check_request(camera, voxel, rotations, clusters, params, max_clusters, max_candidates):
    """Raises ValueError where dsm_viewpoint_enqueue returns DSM_E_INVALID."""
    c = G.Camera(*camera)
    R, v = np.float64(np.float32(c.max_range)), G._v(voxel)
    fin = np.isfinite
    if not (fin(c.fx) and c.fx > 0 and fin(c.fy) and c.fy > 0 and fin(c.cx) and fin(c.cy)):
        raise ValueError("fx, fy must be finite and > 0, cx, cy finite")
    if not (1 <= c.width <= 65536 and 1 <= c.height <= 65536) or c.unknown_blocks not in (0, 1):
        raise ValueError("image size or blocking rule")
    if not (fin(R) and R > 0 and R <= G.MAX_RANGE_VOXELS * v):
        raise ValueError("max_range must be finite, > 0 and at most 128 voxels")
    rot = np.asarray(rotations, np.float64).reshape(-1, 9)
    if not (1 <= len(rot) <= MAX_ROTATIONS) or not fin(rot).all():
        raise ValueError("n_rotations outside [1, 64] or a rotation entry not finite")
    cl = np.asarray(clusters, np.int64).reshape(-1)
    if not (0 <= len(cl) <= max_clusters) or (cl < 0).any():
        raise ValueError("n_clusters outside [0, max_clusters] or a cluster index below 0")
    p = Params(*params)
    if not (0 <= p.r_min <= p.r_max <= MAX_RADIUS and 0 <= p.dz_max <= MAX_DZ and 1 <= p.stride <= MAX_STRIDE):
        raise ValueError("r_min, r_max, dz_max or stride out of range")
    if not (1 <= p.max_samples <= MAX_SAMPLES and p.min_seen >= 0 and 1 <= p.top_k <= MAX_TOP_K and p.with_reach in (0, 1)):
        raise ValueError("max_samples, min_seen, top_k or with_reach out of range")
    if not (fin(np.float32(p.radius)) and np.float32(p.radius) >= 0):
        raise ValueError("radius must be finite and >= 0")
    n_off = len(offsets(p))
    if not (1 <= n_off <= MAX_OFFSETS):
        raise ValueError("n_offsets outside [1, 4096]")
    if len(cl) * n_off > max_candidates:
        raise ValueError("n_clusters n_offsets above max_candidates")
    if len(cl) * n_off * p.max_samples > MAX_WORK:
        raise ValueError("the work bound n_clusters n_offsets max_samples exceeds 2^31 walks")


def centre_voxel(centroid, origin, voxel):
    """int64 (3,): floor(centroid_k / v) - o_k, reach's start snap of the fp64 centroid."""
    return (np.floor(np.asarray(centroid, np.float64) / G._v(voxel)) - np.asarray(origin, np.int64).astype(np.float64)).astype(np.int64)


def sample_positions(n, max_samples):
    """int64 (n_s,): the list positions floor(k n / n_s) of the samples of n listed members."""
    n_s = min(n, max_samples)
    return np.arange(n_s, dtype=np.int64) * n // n_s


def seen_counts(state, origin, voxel, camera, rotations, t, c):
    """int64 (n_rotations,): per rotation r, the centres c (n, 3) in the frustum of [R_r | t] whose walk from t reaches
    them (gain's two tests)."""
    rot = np.asarray(rotations, np.float64).reshape(-1, 3, 3)
    if len(c) == 0:
        return np.zeros(len(rot), np.int64)
    s = G.seen(state, origin, voxel, t, c, G.Camera(*camera).unknown_blocks)
    out = np.zeros(len(rot), np.int64)
    for r, R in enumerate(rot):
        pose = np.concatenate([R, np.asarray(t, np.float64)[:, None]], axis=1).reshape(12)
        out[r] = (G.frustum(c, pose, camera) & s).sum()
    return out


def viewpoints(state, dist, origin, voxel, camera, rotations, clusters, params, frontier, reach_cost=None):
    """(info INFO_DTYPE record, records CLUSTER_DTYPE (n,), slots VIEWPOINT_DTYPE (n, top_k)) of the job on the state
    and fp32 distance grids [nz][ny][nx] at integer origin (x, y, z); frontier: (table, voxel list) of the latest
    frontier job; reach_cost: the latest reach job's uint32 cost grid (needed with with_reach)."""
    p = Params(*params)
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    shape = np.array([nx, ny, nz], np.int64)
    table, vox = frontier
    rot = np.asarray(rotations, np.float64).reshape(-1, 9)
    cl = np.asarray(clusters, np.int64).reshape(-1)
    off = offsets(p)
    trav = pyoracle_reach.traversable(st, dist, p.radius)
    recs = np.zeros(len(cl), CLUSTER_DTYPE)
    slots = np.zeros((len(cl), p.top_k), VIEWPOINT_DTYPE)
    slots["voxel"], slots["offset"], slots["rotation"], slots["cost"] = -1, -1, -1, INF
    for i, c in enumerate(cl):
        r = recs[i]
        r["cluster"] = c
        past = c >= len(table)
        r["status"] = 3 if past else 2 if table[c]["offset"] < 0 else 0
        if r["status"]:
            continue
        T = table[c]
        g = centre_voxel(T["centroid"], origin, voxel)
        members = vox[T["offset"]:T["offset"] + T["n_voxels"]].astype(np.int64)
        m = members[sample_positions(len(members), p.max_samples)]
        r["n_samples"] = len(m)
        mc = G.centres(np.stack([m % nx, m // nx % ny, m // (nx * ny)], 1), origin, voxel)
        cand = g + off
        inside = ((cand >= 0) & (cand < shape)).all(axis=1)
        r["n_inside"] = inside.sum()
        ranked = []
        for j in np.flatnonzero(inside):
            x, y, z = cand[j]
            if not trav[z, y, x]:
                continue
            r["n_traversable"] += 1
            cost = INF
            if p.with_reach:
                cost = int(reach_cost[z, y, x])
                if cost == INF:
                    continue
            r["n_reached"] += 1
            t = G.centres([cand[j]], origin, voxel)[0]
            seen = seen_counts(st, origin, voxel, camera, rot, t, mc)
            best = int(np.argmax(seen))      # the first maximum: the lowest rotation on ties
            n_seen = int(seen[best])
            if n_seen >= max(1, p.min_seen):
                ranked.append((-n_seen, cost, int(j), best, int((z * ny + y) * nx + x)))
        ranked.sort()
        for k, (neg, cost, j, best, lin) in enumerate(ranked[:p.top_k]):
            slots[i, k] = (lin, j, best, -neg, cost, (0, 0, 0))
        r["n_viewpoints"] = min(len(ranked), p.top_k)
    info = np.zeros((), INFO_DTYPE)
    info["origin"] = np.asarray(origin, np.int32)
    info["n_clusters"], info["n_offsets"], info["n_rotations"], info["top_k"] = len(cl), len(off), len(rot), p.top_k
    info["unknown_blocks"], info["with_reach"], info["n_clusters_table"] = G.Camera(*camera).unknown_blocks, p.with_reach, len(table)
    return info, recs, slots
