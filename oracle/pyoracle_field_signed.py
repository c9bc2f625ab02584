"""The signed distance field of dsm_field_signed_enable (DESIGN.md §8.16, include/dsm.h) restated in numpy: dist on the
voxels F that are not sites, (1 - sqrtf((float)e2)) * v on the sites S (e2 the squared integer distance to F), the
+-INFINITY rules, and the signed queries, on the fields of oracle/pyoracle_field and oracle/pyoracle_field_known."""
import numpy as np

import pyoracle_field
import pyoracle_field_known
import pyoracle_field_query


def signed(sites, dist, voxel):
    """float32 [nz][ny][nx] sdist of the bool site mask `sites` whose distance grid is `dist` (float32, same shape)."""
    sites = np.asarray(sites, bool)
    dist = np.asarray(dist, np.float32)
    if sites.all():
        return np.full(sites.shape, -np.inf, np.float32)
    if not sites.any():
        return dist.copy()
    e2 = pyoracle_field.squared_distances(~sites)   # to the nearest voxel of F; 0 exactly on F
    depth = (np.float32(1) - np.sqrt(e2.astype(np.float32))) * np.float32(voxel)
    return np.where(sites, depth, dist).astype(np.float32)


def field(points, voxel, shape, center):
    """(dist, sdist, origin, n_occupied) of a plain request, as pyoracle_field.field; the sites are the occupied voxels."""
    dist, o, n_occ = pyoracle_field.field(points, voxel, shape, center)
    pts = np.asarray(points, np.float32)
    pts = pts.reshape(len(pts), -1)[:, :3] if pts.size else np.zeros((0, 3), np.float32)
    occ = pyoracle_field.occupancy(pts, voxel, shape, o.astype(np.int64))
    return dist, signed(occ, dist, voxel), o, n_occ


def state_field(state, voxel):
    """(dist, sdist) of a state grid [nz][ny][nx] (0 unknown, 1 occupied, 2 free); the sites are the voxels that are not
    free."""
    dist = pyoracle_field_known.state_field(state, voxel)[0]
    return dist, signed(np.asarray(state) != pyoracle_field_known.FREE, dist, voxel)


def sample(sdist, origin, voxel, points):
    """pyoracle_field_query.sample on the signed grid, with its two rules: no site (every voxel +inf) gives +inf, no voxel
    of F (every voxel -inf) gives -inf, both with a zero gradient."""
    sdist = np.asarray(sdist, np.float32)
    if not np.isneginf(sdist).all():
        return pyoracle_field_query.sample(sdist, origin, voxel, points)   # finite everywhere, or +inf everywhere
    out = pyoracle_field_query.sample(np.full(sdist.shape, np.inf, np.float32), origin, voxel, points)
    out["dist"][out["dist"] == np.inf] = -np.inf
    return out


def clearance(sdist, origin, voxel, waypoints, offsets, step, radius):
    """pyoracle_field_query.clearance on the signed grid: the same samples and reductions over sample()'s distances."""
    wp, ofs = pyoracle_field_query.check_request(waypoints, offsets, step, radius)
    pts, traj, idx = pyoracle_field_query.trajectory_samples(wp, ofs, step)
    n = len(ofs) - 1
    out = np.zeros(n, pyoracle_field_query.CLEARANCE_DTYPE)
    if n == 0:
        return out
    d = sample(sdist, origin, voxel, pts)["dist"]
    inside = ~np.isnan(d)
    starts = np.concatenate([[0], np.cumsum(np.bincount(traj, minlength=n))[:-1]])
    big = np.iinfo(np.int64).max
    mind = np.minimum.reduceat(np.where(inside, d, np.float32(np.inf)), starts).astype(np.float32)
    arg = np.minimum.reduceat(np.where(inside & (d == mind[traj]), idx, big), starts)
    hit = np.minimum.reduceat(np.where(inside & (d < np.float32(radius)), idx, big), starts)
    out["min_dist"] = mind
    out["argmin"] = np.where(arg == big, -1, arg)
    out["first_hit"] = np.where(hit == big, -1, hit)
    out["n_outside"] = np.add.reduceat((~inside).astype(np.int64), starts)
    return out
