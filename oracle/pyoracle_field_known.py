"""The known-space field of dsm_field_enqueue_known (DESIGN.md §8.9) restated in numpy: the rays a capture keeps, the
fp64 Amanatides-Woo walk of every ray (all rays of a call in lockstep), the three-state grid and the distance to the
nearest voxel that is not known to be free, built on pyoracle_field's occupancy and exact EDT."""
import numpy as np

import pyoracle_field

UNKNOWN, OCCUPIED, FREE = 0, 1, 2
VIEWS_MAX = 65536


def capture(seeds):
    """The rays dsm_views_capture keeps of one frame's SEED_DTYPE records, in seed index order: float32 (n, 3) posi of
    every seed with mean_depth > 0 and three finite coordinates."""
    p = np.stack([seeds["posi_x"], seeds["posi_y"], seeds["posi_z"]], axis=1).astype(np.float32)
    with np.errstate(invalid="ignore"):
        keep = (seeds["mean_depth"] > 0) & np.isfinite(p).all(axis=1)
    return p[keep]


def check_enable(max_views, max_range, voxel):
    """Raises ValueError where dsm_views_enable returns DSM_E_INVALID."""
    r = np.float32(max_range)
    if not (1 <= max_views <= VIEWS_MAX):
        raise ValueError("max_views outside [1, 65536]")
    if not (np.isfinite(r) and r > 0 and np.float64(r) <= 1024.0 * np.float64(np.float32(voxel))):
        raise ValueError("max_range must be finite, > 0 and at most 1024 voxels")


def segments(rays, pose, max_range):
    """(a, b, truncated) of the rays (n, 3) float32 of one view at pose (12,) row-major [R | t] (camera to world):
    a = t and b the ray's end in fp64, cut to max_range when longer (truncated)."""
    P = np.asarray(pose, np.float64).reshape(3, 4)
    p = np.asarray(rays, np.float32).reshape(-1, 3).astype(np.float64)
    t = P[:, 3]
    with np.errstate(over="ignore", invalid="ignore"):   # R * p may overflow: see walk for such rays
        b = ((P[:, 0] * p[:, :1] + P[:, 1] * p[:, 1:2]) + P[:, 2] * p[:, 2:3]) + t
        a = np.broadcast_to(t, b.shape).copy()
        d = b - a
        L = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        mr = np.float64(np.float32(max_range))
        trunc = L > mr
        f = mr / L[trunc]
        b[trunc] = a[trunc] + f[:, None] * d[trunc]
    return a, b, trunc


def walk(a, b, voxel, visit=None):
    """Every visit of the walk of include/dsm.h from a to b (n, 3) fp64, all rays in lockstep: (ray, voxel (m, 3) int64,
    end (m,) bool: the visit is the end voxel e).  Rays with a non-finite endpoint visit nothing.  With `visit`, each
    step's visits go to visit(ray, voxel, end) instead, and nothing is returned."""
    v = np.float64(np.float32(voxel))
    a = np.asarray(a, np.float64).reshape(-1, 3)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        wa, wb = a / v, b / v
        ok = np.isfinite(wa).all(axis=1) & np.isfinite(wb).all(axis=1)
        rid = np.nonzero(ok)[0]
        wa, wb = wa[ok], wb[ok]
        i, e = np.floor(wa), np.floor(wb)   # integers, exact in fp64
        delta = wb - wa
        s = np.sign(delta)
        tD = np.where(delta != 0, 1.0 / np.abs(delta), np.inf)
        tM = np.where(delta > 0, ((i + 1) - wa) / delta, np.where(delta < 0, (i - wa) / delta, np.inf))
    out_r, out_v, out_e = [], [], []
    act = np.arange(len(rid))
    while len(act):
        end = (i[act] == e[act]).all(axis=1)
        if visit is None:
            out_r.append(rid[act])
            out_v.append(i[act].astype(np.int64))
            out_e.append(end)
        else:
            visit(rid[act], i[act].astype(np.int64), end)
        act = act[~end]
        k = np.argmin(tM[act], axis=1)     # the first minimum: the lowest axis on ties
        tk = tM[act, k]
        act, k = act[tk <= 1.0], k[tk <= 1.0]
        i[act, k] += s[act, k]
        tM[act, k] = tM[act, k] + tD[act, k]
    if visit is not None:
        return None
    if not out_r:
        return np.zeros(0, np.int64), np.zeros((0, 3), np.int64), np.zeros(0, bool)
    return np.concatenate(out_r), np.concatenate(out_v), np.concatenate(out_e)


def carve(state, views, voxel, o, max_range, batch=1 << 17):
    """Stores FREE into every UNKNOWN voxel of state [nz][ny][nx] (uint8, in place) that a ray of views [(rays, pose)]
    visits, except the end voxel of a ray that was not truncated.  Carving only turns UNKNOWN into FREE, so the views
    are walked in batches of about `batch` rays, in any order."""
    nz, ny, nx = state.shape
    o = np.asarray(o, np.int64)
    n = np.array([nx, ny, nz], np.int64)

    def flush(segs):
        a = np.concatenate([x[0] for x in segs])
        b = np.concatenate([x[1] for x in segs])
        trunc = np.concatenate([x[2] for x in segs])

        def visit(r, ijk, end):
            q = ijk - o
            keep = (q >= 0).all(axis=1) & (q < n).all(axis=1) & ~(end & ~trunc[r])
            q = q[keep]
            cell = state[q[:, 2], q[:, 1], q[:, 0]]
            q = q[cell == UNKNOWN]
            state[q[:, 2], q[:, 1], q[:, 0]] = FREE
        walk(a, b, voxel, visit)

    segs, count = [], 0
    for rays, pose in views:
        segs.append(segments(rays, pose, max_range))
        count += len(segs[-1][0])
        if count >= batch:
            flush(segs)
            segs, count = [], 0
    if segs:
        flush(segs)
    return state


def known_field(points, voxel, shape, center, views, max_range):
    """(dist, origin, n_occupied, state, n_free) of a known request centred on `center` over the obstacle points (as
    pyoracle_field.field) and the views [(rays (n, 3) float32, pose (12,) fp64)].  Raises ValueError where the library
    returns DSM_E_INVALID for the centre or a pose."""
    o = pyoracle_field.origin(center, voxel, shape)
    if o is None:
        raise ValueError("origin outside +-2^24 voxels")
    for _, pose in views:
        if not np.isfinite(np.asarray(pose, np.float64)).all() or np.size(pose) != 12:
            raise ValueError("a pose entry is not finite")
    pts = np.asarray(points, np.float32)
    pts = pts.reshape(len(pts), -1)[:, :3] if pts.size else np.zeros((0, 3), np.float32)
    state = pyoracle_field.occupancy(pts, voxel, shape, o).astype(np.uint8)
    carve(state, views, voxel, o, max_range)
    dist, n_occupied, n_free = state_field(state, voxel)
    return dist, o.astype(np.int32), n_occupied, state, n_free


def state_field(state, voxel):
    """(dist, n_occupied, n_free) of the state grid [nz][ny][nx] (uint8): the distance to the nearest voxel that is not
    free (float32, +inf when every voxel is free), the occupied and the free voxels."""
    d2 = pyoracle_field.squared_distances(state != FREE)
    if d2 is None:
        dist = np.full(state.shape, np.inf, np.float32)
    else:
        dist = np.sqrt(d2.astype(np.float32)) * np.float32(voxel)
    return dist.astype(np.float32), int((state == OCCUPIED).sum()), int((state == FREE).sum())
