"""The distance field of dsm_field_enqueue (DESIGN.md §8.7) restated in numpy: the grid origin, the occupancy of the
obstacle points and the exact Euclidean distance transform, through scipy's exact EDT."""
import numpy as np
from scipy import ndimage

LIMIT = 1 << 24  # |o_k| and |o_k + n_k| bound: the fp32 compares below are exact under it


def origin(center, voxel, shape):
    """o_k = floor(c_k / (double)v) - floor(n_k / 2) in int64, (x, y, z); shape = (nx, ny, nz).  None when it breaks the
    2^24 bound (the library returns DSM_E_INVALID)."""
    v = np.float64(np.float32(voxel))
    n = np.asarray(shape, np.int64)
    q = np.floor(np.asarray(center, np.float64) / v)
    if not np.all(np.abs(q) <= 4.0 * LIMIT):
        return None
    o = q.astype(np.int64) - n // 2
    if np.any(np.abs(o) > LIMIT) or np.any(np.abs(o + n) > LIMIT):
        return None
    return o


def occupancy(points, voxel, shape, o):
    """[nz][ny][nx] bool: voxel q - o of every point with o_k <= q_k < o_k + n_k, q = floor(float32(p) / float32(v))."""
    nx, ny, nz = shape
    p = np.asarray(points, np.float32).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        q = np.floor(p / np.float32(voxel))
        lo = np.asarray(o, np.int64).astype(np.float32)
        hi = (np.asarray(o, np.int64) + np.asarray(shape, np.int64)).astype(np.float32)
        inside = np.all((q >= lo) & (q < hi), axis=1)
    idx = q[inside].astype(np.int64) - np.asarray(o, np.int64)
    occ = np.zeros((nz, ny, nx), bool)
    occ[idx[:, 2], idx[:, 1], idx[:, 0]] = True
    return occ


def squared_distances(occ):
    """int64 d2 per voxel: the smallest squared integer distance to an occupied voxel (None when none is occupied)."""
    if not occ.any():
        return None
    _, ind = ndimage.distance_transform_edt(~occ, return_indices=True)
    d2 = np.zeros(occ.shape, np.int64)
    for k, n in enumerate(occ.shape):   # one axis at a time: the peak stays near the index array's size
        shape = [1] * occ.ndim
        shape[k] = n
        diff = ind[k].astype(np.int64) - np.arange(n, dtype=np.int64).reshape(shape)
        d2 += diff * diff
    return d2


def field(points, voxel, shape, center):
    """(dist, origin, n_occupied) of a request centred on `center` over the obstacle points (n, 3) (or (n, 4) PointXYZI,
    whose fourth column is ignored); dist float32 [nz][ny][nx], origin int32 (x, y, z).  Raises ValueError where the
    library returns DSM_E_INVALID."""
    o = origin(center, voxel, shape)
    if o is None:
        raise ValueError("origin outside +-2^24 voxels")
    pts = np.asarray(points, np.float32)
    pts = pts.reshape(len(pts), -1)[:, :3] if pts.size else np.zeros((0, 3), np.float32)
    occ = occupancy(pts, voxel, shape, o)
    d2 = squared_distances(occ)
    if d2 is None:
        dist = np.full(occ.shape, np.inf, np.float32)
    else:
        dist = np.sqrt(d2.astype(np.float32)) * np.float32(voxel)
    return dist.astype(np.float32), o.astype(np.int32), int(occ.sum())
