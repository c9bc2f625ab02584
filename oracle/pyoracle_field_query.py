"""The planner queries of dsm_field_query_* (DESIGN.md §8.8, include/dsm.h) restated in numpy: the trilinear point query
with its gradient and the trajectory clearance, on a distance field of oracle/pyoracle_field.  Addressing and sampling
are float64, the interpolation float32 with one rounding per operation, as the library computes them (it is built with
-fmad=false), so the restatement is bit for bit."""
import numpy as np

MAX_SAMPLES = 1 << 26   # trajectory samples one call may ask for
QNAN = np.array([0x7FC00000], np.uint32).view(np.float32)[0]   # the canonical quiet NaN: outside the grid
SAMPLE_DTYPE = np.dtype([("dist", "<f4"), ("gx", "<f4"), ("gy", "<f4"), ("gz", "<f4")])
CLEARANCE_DTYPE = np.dtype([("min_dist", "<f4"), ("argmin", "<i4"), ("first_hit", "<i4"), ("n_outside", "<i4")])


def _axis(p, v, o, n):
    """(inside, i, j, t) of one axis: u = p / v - o - 0.5 in float64; inside when 0 <= u <= n - 1."""
    with np.errstate(invalid="ignore", over="ignore"):
        u = p / v - np.float64(o) - 0.5
        inside = (u >= 0.0) & (u <= np.float64(n - 1))
    i = np.minimum(np.floor(np.where(inside, u, 0.0)), max(n - 2, 0)).astype(np.int64)
    j = np.minimum(i + 1, n - 1)
    t = np.where(inside, u - i, 0.0).astype(np.float32)
    return inside, i, j, t


def _lerp(a, b, t):
    return a + t * (b - a)   # float32 arrays: one rounding per operation


def sample(dist, origin, voxel, points):
    """SAMPLE_DTYPE (n,) of the point query at points (n, 3) on the field dist (float32 [nz][ny][nx]) with origin
    (x, y, z) in voxels and voxel edge `voxel` (taken as float32)."""
    dist = np.asarray(dist, np.float32)
    nz, ny, nx = dist.shape
    p = np.asarray(points, np.float64).reshape(-1, 3)
    v32 = np.float32(voxel)
    v = np.float64(v32)
    ax = [_axis(p[:, k], v, int(origin[k]), n) for k, n in enumerate((nx, ny, nz))]
    inside = ax[0][0] & ax[1][0] & ax[2][0]
    (_, ix, jx, tx), (_, iy, jy, ty), (_, iz, jz, tz) = ax
    out = np.zeros(len(p), SAMPLE_DTYPE)
    out["dist"] = QNAN
    empty = not np.isfinite(dist).any()   # a field with an occupied voxel is finite everywhere
    if empty:
        out["dist"][inside] = np.inf
        return out
    c = {}
    for kz, z in (("0", iz), ("1", jz)):
        for ky, y in (("0", iy), ("1", jy)):
            for kx, x in (("0", ix), ("1", jx)):
                c[kx + ky + kz] = dist[z, y, x]
    d = _lerp(_lerp(_lerp(c["000"], c["100"], tx), _lerp(c["010"], c["110"], tx), ty),
              _lerp(_lerp(c["001"], c["101"], tx), _lerp(c["011"], c["111"], tx), ty), tz)
    gx = _lerp(_lerp(c["100"] - c["000"], c["110"] - c["010"], ty), _lerp(c["101"] - c["001"], c["111"] - c["011"], ty), tz) / v32
    gy = _lerp(_lerp(c["010"] - c["000"], c["110"] - c["100"], tx), _lerp(c["011"] - c["001"], c["111"] - c["101"], tx), tz) / v32
    gz = _lerp(_lerp(c["001"] - c["000"], c["101"] - c["100"], tx), _lerp(c["011"] - c["010"], c["111"] - c["110"], tx), ty) / v32
    for name, val in (("dist", d), ("gx", gx), ("gy", gy), ("gz", gz)):
        out[name][inside] = val[inside]
    return out


def check_request(waypoints, offsets, step, radius):
    """(waypoints (w, 3) float64, offsets int64) of a valid trajectory request; ValueError where the library returns
    DSM_E_INVALID (capacities aside): offsets not starting at 0 or not rising strictly, offsets[-1] beyond the
    waypoints, a non-finite waypoint, step not finite and > 0, radius not finite and >= 0, more than 2^26 samples."""
    wp = np.asarray(waypoints, np.float64).reshape(-1, 3)
    ofs = np.asarray(offsets, np.int64).reshape(-1)
    step, radius = np.float32(step), np.float32(radius)
    if not (np.isfinite(step) and step > 0) or not (np.isfinite(radius) and radius >= 0):
        raise ValueError("step must be finite and > 0, radius finite and >= 0")
    if len(ofs) < 1 or ofs[0] != 0 or np.any(np.diff(ofs) <= 0) or ofs[-1] > len(wp):
        raise ValueError("offsets must start at 0 and rise strictly within the waypoints")
    wp = wp[:ofs[-1]]
    if not np.isfinite(wp).all():
        raise ValueError("non-finite waypoint")
    return wp, ofs


def segment_counts(wp, ofs, step):
    """Samples per waypoint: m = max(1, ceil(L / step)) for the segment it starts, 1 for a trajectory's last waypoint;
    ValueError above 2^26 in all."""
    last = np.zeros(len(wp), bool)
    last[ofs[1:] - 1] = True
    nxt = np.minimum(np.arange(len(wp)) + 1, max(len(wp) - 1, 0))
    with np.errstate(invalid="ignore", over="ignore"):
        d = wp[nxt] - wp
        L = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        m = np.where(last, 1.0, np.maximum(1.0, np.ceil(L / np.float64(np.float32(step)))))
    if not np.isfinite(m).all() or m.sum() > MAX_SAMPLES:
        raise ValueError("more than 2^26 trajectory samples")
    return m.astype(np.int64), nxt, last


def trajectory_samples(waypoints, offsets, step):
    """(points (S, 3) float64, trajectory of each sample, its index along the trajectory) of every trajectory, in order."""
    wp, ofs = check_request(waypoints, offsets, step, 0.0)
    m, nxt, last = segment_counts(wp, ofs, step)
    seg = np.repeat(np.arange(len(wp)), m)
    start = np.cumsum(m) - m                      # global index of each waypoint's first sample
    k = np.arange(len(seg)) - start[seg]          # index within the segment
    f = k / m[seg].astype(np.float64)
    a, b = wp[seg], wp[nxt[seg]]
    pts = np.where(last[seg][:, None], a, a + f[:, None] * (b - a))
    traj = np.repeat(np.arange(len(ofs) - 1), np.add.reduceat(m, ofs[:-1]) if len(ofs) > 1 else np.zeros(0, np.int64))
    tstart = (np.cumsum(m) - m)[ofs[:-1]] if len(ofs) > 1 else np.zeros(0, np.int64)
    return pts, traj, np.arange(len(seg)) - tstart[traj]


def clearance(dist, origin, voxel, waypoints, offsets, step, radius):
    """CLEARANCE_DTYPE (t,) of the trajectories (waypoints (w, 3), offsets (t + 1,)) sampled at `step`, against
    `radius` (both taken as float32), on the field dist with origin and voxel as in sample()."""
    wp, ofs = check_request(waypoints, offsets, step, radius)
    pts, traj, idx = trajectory_samples(wp, ofs, step)
    n = len(ofs) - 1
    out = np.zeros(n, CLEARANCE_DTYPE)
    if n == 0:
        return out
    d = sample(dist, origin, voxel, pts)["dist"]
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
