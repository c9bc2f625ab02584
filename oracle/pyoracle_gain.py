"""The view gain of dsm_gain_enqueue (DESIGN.md §8.12) restated in numpy: per camera pose, the frustum voxels of a known
field's state grid and the free, unknown, occupied, frontier and cluster voxels seen through it along the fp64
Amanatides-Woo walk of dsm_field_enqueue_known (pyoracle_field_known.walk), with the records and the header in the
layout dsm_gain_wait hands out.  The host's per-view box is restated too, so that a test can show it never cuts a
counted voxel."""
from collections import namedtuple

import numpy as np

import pyoracle_frontier

UNKNOWN, OCCUPIED, FREE = 0, 1, 2
MAX_VIEWS = 1 << 20          # DSM_GAIN_MAX_VIEWS
MAX_RANGE_VOXELS = 128       # DSM_GAIN_MAX_RANGE_VOXELS
MAX_WORK = 1 << 31           # DSM_GAIN_MAX_WORK
ORTHONORMAL_TOL = 1e-6       # the box uses the image pyramid only for a pose this close to a rotation

GAIN_DTYPE = np.dtype([("n_frustum", "<i4"), ("n_free", "<i4"), ("n_unknown", "<i4"), ("n_occupied", "<i4"), ("n_frontier", "<i4"),
                       ("n_cluster", "<i4"), ("status", "<i4"), ("reserved", "<i4")])
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_views", "<i4"), ("n_clusters_table", "<i4"), ("unknown_blocks", "<i4"),
                       ("reserved", "<i4", 2)])

Camera = namedtuple("Camera", "fx fy cx cy width height max_range unknown_blocks")


def _v(voxel):
    return np.float64(np.float32(voxel))


def check_enable(max_views):
    """Raises ValueError where dsm_gain_enable returns DSM_E_INVALID."""
    if not (1 <= max_views <= MAX_VIEWS):
        raise ValueError("max_views outside [1, 2^20]")


def check_request(camera, voxel, poses, clusters, max_views):
    """Raises ValueError where dsm_gain_enqueue returns DSM_E_INVALID."""
    c = Camera(*camera)
    fin = np.isfinite
    if not (fin(c.fx) and c.fx > 0 and fin(c.fy) and c.fy > 0 and fin(c.cx) and fin(c.cy)):
        raise ValueError("fx, fy must be finite and > 0, cx, cy finite")
    if not (1 <= c.width <= 65536 and 1 <= c.height <= 65536):
        raise ValueError("width or height outside [1, 65536]")
    if c.unknown_blocks not in (0, 1):
        raise ValueError("unknown_blocks must be 0 or 1")
    R, v = np.float64(np.float32(c.max_range)), _v(voxel)
    if not (fin(R) and R > 0 and R <= MAX_RANGE_VOXELS * v):
        raise ValueError("max_range must be finite, > 0 and at most 128 voxels")
    P = np.asarray(poses, np.float64).reshape(-1, 12)
    if not (0 <= len(P) <= max_views):
        raise ValueError("n_views outside [0, max_views]")
    m = 2 * int(np.ceil(R / v)) + 3
    if len(P) * m ** 3 > MAX_WORK:
        raise ValueError("the work bound n_views (2 ceil(R / v) + 3)^3 exceeds 2^31 voxels")
    if not np.isfinite(P).all():
        raise ValueError("a pose entry is not finite")
    if clusters is not None and (np.asarray(clusters) < -1).any():
        raise ValueError("a cluster index below -1")


def centres(xyz, origin, voxel):
    """fp64 world centres ((o + x) + 0.5) v of grid voxels xyz (n, 3)."""
    return ((np.asarray(origin, np.int64) + np.asarray(xyz, np.int64)).astype(np.float64) + 0.5) * _v(voxel)


def frustum(c, pose, camera):
    """bool (n,): the centres c (n, 3) fp64 that pass the frustum test of view `pose` (12,)."""
    cam = Camera(*camera)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    d = c - P[:, 3]
    R = np.float64(np.float32(cam.max_range))
    r2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    q = [(P[0, m] * d[:, 0] + P[1, m] * d[:, 1]) + P[2, m] * d[:, 2] for m in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = np.float64(cam.fx) * (q[0] / q[2]) + np.float64(cam.cx)
        w = np.float64(cam.fy) * (q[1] / q[2]) + np.float64(cam.cy)
        return ((r2 <= R * R) & (q[2] > 0) & (u >= 0) & (u < np.float64(cam.width)) & (w >= 0) &
                (w < np.float64(cam.height)))


def box(pose, camera, voxel, origin, shape, pyramid=True):
    """(lo, size) int64 (3,) in grid coordinates: the host's box of view `pose` on a grid of shape (nx, ny, nz).  The
    bounding box of the apex and the four image corners at depth max_range, met with the cube around the range sphere
    (the cube alone with pyramid=False, for a pose that is no rotation, or for a corner that is not finite), padded by
    one voxel and clipped to the grid; size 0 on an axis when empty."""
    cam = Camera(*camera)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    t = P[:, 3]
    R, v = np.float64(np.float32(cam.max_range)), _v(voxel)
    use = pyramid
    for a in range(3):
        for b in range(3):
            s = (P[0, a] * P[0, b] + P[1, a] * P[1, b]) + P[2, a] * P[2, b]
            use = use and abs(s - (1.0 if a == b else 0.0)) <= ORTHONORMAL_TOL
    plo, phi = t.copy(), t.copy()
    with np.errstate(over="ignore", invalid="ignore"):
        for uu in (0.0, np.float64(cam.width)):
            for ww in (0.0, np.float64(cam.height)):
                qx = ((uu - np.float64(cam.cx)) / np.float64(cam.fx)) * R
                qy = ((ww - np.float64(cam.cy)) / np.float64(cam.fy)) * R
                p = ((P[:, 0] * qx + P[:, 1] * qy) + P[:, 2] * R) + t
                use = use and bool(np.isfinite(p).all())
                plo, phi = np.minimum(plo, p), np.maximum(phi, p)
    lo, hi = t - R, t + R
    if use:
        lo, hi = np.maximum(lo, plo), np.minimum(hi, phi)
    o = np.asarray(origin, np.int64).astype(np.float64)
    n = np.asarray(shape, np.int64)
    a = np.maximum(np.floor(lo / v) - 1.0 - o, 0.0)
    b = np.minimum(np.floor(hi / v) + 1.0 - o, (n - 1).astype(np.float64))
    ok = a <= b
    if not ok.all():
        return np.zeros(3, np.int64), np.zeros(3, np.int64)
    return a.astype(np.int64), (b - a).astype(np.int64) + 1


def seen(state, origin, voxel, t, c, unknown_blocks):
    """bool (n,): the walks of include/dsm.h from t (3,) to the centres c (n, 3), all in lockstep, that reach their end
    voxel with every voxel before it inside the grid and passing the blocking rule.  A walk leaves at its first blocking
    voxel; pyoracle_field_known.walk, which runs every walk to its end, gives the same answers (tests/test_gain_model.py)."""
    st = np.asarray(state)
    nz, ny, nx = st.shape
    n = np.array([nx, ny, nz], np.int64)
    o = np.asarray(origin, np.int64)
    v = _v(voxel)
    c = np.asarray(c, np.float64).reshape(-1, 3)
    wa = np.broadcast_to(np.asarray(t, np.float64) / v, c.shape)
    wb = c / v
    i, e = np.floor(wa), np.floor(wb)
    with np.errstate(divide="ignore", invalid="ignore"):
        delta = wb - wa
        s = np.sign(delta)
        tD = np.where(delta != 0, 1.0 / np.abs(delta), np.inf)
        tM = np.where(delta > 0, ((i + 1) - wa) / delta, np.where(delta < 0, (i - wa) / delta, np.inf))
    i = i.copy()
    out = np.zeros(len(c), bool)
    act = np.arange(len(c))
    while len(act):
        end = (i[act] == e[act]).all(axis=1)
        out[act[end]] = True
        act = act[~end]
        q = i[act].astype(np.int64) - o
        inside = (q >= 0).all(axis=1) & (q < n).all(axis=1)
        act, q = act[inside], q[inside]
        cell = st[q[:, 2], q[:, 1], q[:, 0]]
        act = act[cell == FREE] if unknown_blocks else act[cell != OCCUPIED]
        k = np.argmin(tM[act], axis=1)      # the first minimum: the lowest axis on ties
        tk = tM[act, k]
        act, k = act[tk <= 1.0], k[tk <= 1.0]
        i[act, k] += s[act, k]
        tM[act, k] = tM[act, k] + tD[act, k]
    return out


def cluster_slots(shape_zyx, table, vox):
    """int32 [nz][ny][nx]: the table entry whose listed voxels hold each voxel, -1 elsewhere."""
    slot = np.full(int(np.prod(shape_zyx)), -1, np.int32)
    for ci, rec in enumerate(table):
        if rec["offset"] >= 0:
            slot[vox[rec["offset"]:rec["offset"] + rec["n_voxels"]]] = ci
    return slot.reshape(shape_zyx)


def camera_inside(pose, voxel, origin, shape):
    t = np.asarray(pose, np.float64).reshape(3, 4)[:, 3]
    q = np.floor(t / _v(voxel)) - np.asarray(origin, np.int64).astype(np.float64)
    return bool(((q >= 0) & (q < np.asarray(shape, np.float64))).all())


def gains(state, origin, voxel, camera, poses, clusters=None, frontier=None, pyramid=True):
    """(info INFO_DTYPE record, records GAIN_DTYPE (n_views,)) of the views poses (n, 12) on the state grid [nz][ny][nx]
    at integer origin (x, y, z).  clusters: n table indices (-1: none) or None; frontier: (table, voxel list) of the
    latest frontier job (needed with clusters).  pyramid=False enumerates the whole padded cube of the range sphere
    instead of the host's box, which the counts must not notice."""
    cam = Camera(*camera)
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    shape = (nx, ny, nz)
    P = np.asarray(poses, np.float64).reshape(-1, 12)
    front = pyoracle_frontier.frontier_mask(st)
    table, vox = frontier if frontier is not None else (np.zeros(0, pyoracle_frontier.CLUSTER_DTYPE), np.zeros(0, np.int32))
    n_table = len(table) if clusters is not None else 0
    slot = cluster_slots(st.shape, table, vox) if clusters is not None else None
    out = np.zeros(len(P), GAIN_DTYPE)
    for j, pose in enumerate(P):
        cl = -1 if clusters is None else int(clusters[j])
        past = cl >= n_table
        unlisted = 0 <= cl < n_table and table[cl]["offset"] < 0
        inside = camera_inside(pose, voxel, origin, shape)
        r = out[j]
        r["status"] = 1 if not inside else 0 if cl < 0 else 3 if past else 2 if unlisted else 0
        r["n_cluster"] = -1 if cl < 0 or past or unlisted else 0
        lo, size = box(pose, cam, voxel, origin, shape, pyramid)
        if (size == 0).any():
            continue
        g = np.stack(np.meshgrid(*[np.arange(lo[k], lo[k] + size[k]) for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
        c = centres(g, origin, voxel)
        f = frustum(c, pose, cam)
        g, c = g[f], c[f]
        r["n_frustum"] = len(g)
        s = seen(st, origin, voxel, pose.reshape(3, 4)[:, 3], c, cam.unknown_blocks)
        g = g[s]
        sv = st[g[:, 2], g[:, 1], g[:, 0]]
        r["n_free"], r["n_unknown"], r["n_occupied"] = (sv == FREE).sum(), (sv == UNKNOWN).sum(), (sv == OCCUPIED).sum()
        r["n_frontier"] = front[g[:, 2], g[:, 1], g[:, 0]].sum()
        if r["n_cluster"] == 0:
            r["n_cluster"] = (slot[g[:, 2], g[:, 1], g[:, 0]] == cl).sum()
    info = np.zeros((), INFO_DTYPE)
    info["origin"] = np.asarray(origin, np.int32)
    info["n_views"], info["n_clusters_table"], info["unknown_blocks"] = len(P), n_table, cam.unknown_blocks
    return info, out
