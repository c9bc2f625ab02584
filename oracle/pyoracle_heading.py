"""The heading job of dsm_heading_* (DESIGN.md §8.19, include/dsm.h) restated in numpy: per sample of uniform cubic
B-spline trajectories (pyoracle_trajectory.curve_samples) and per rotation of a list, the unknown and frontier voxels a
camera there would see (gain's frustum test and walk, pyoracle_gain.frustum and pyoracle_gain.seen, one walk per voxel
for every rotation), then per trajectory the best rate-limited rotation sequence by a backward pass over (sample,
rotation) and a forward trace, with the header and the records in the layout dsm_heading_wait hands out.

The counts are integers and the scores int64, so the restatement is exact; the sample positions are fp64 with one
rounding per operation, as the library evaluates them on the host."""
import numpy as np

import pyoracle_frontier
import pyoracle_gain as G
import pyoracle_trajectory as tj

MAX_ROTATIONS = 64           # DSM_HEADING_MAX_ROTATIONS
MAX_K = 64                   # DSM_HEADING_MAX_SAMPLES_PER_SEGMENT
MAX_WEIGHT = 1 << 16         # DSM_HEADING_MAX_WEIGHT
MAX_CAPACITY = 1 << 22       # DSM_HEADING_MAX_CAPACITY
MAX_WORK = 1 << 31           # DSM_HEADING_MAX_WORK: sum over samples of (2 ceil(R / v) + 3)^3

REQUEST_DTYPE = np.dtype([("start", "<i4"), ("end", "<i4"), ("max_step", "<i4"), ("reserved", "<i4")])
RECORD_DTYPE = np.dtype([("status", "<i4"), ("n_samples", "<i4"), ("sample_offset", "<i4"), ("n_outside", "<i4"), ("score", "<i8"),
                         ("steps", "<i4"), ("reserved", "<i4")])
SAMPLE_DTYPE = np.dtype([("p", "<f8", 3), ("rotation", "<i4"), ("turn", "<i4")])
COUNT_DTYPE = np.dtype([("n_unknown", "<i4"), ("n_frontier", "<i4")])
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_trajectories", "<i4"), ("n_samples", "<i4"), ("n_rot", "<i4"), ("unknown_blocks", "<i4"),
                       ("n_status", "<i4", 2), ("reserved", "<i4", 7)])


def requests(rows):
    """REQUEST_DTYPE (n,) of (start, end, max_step) triples."""
    out = np.zeros(len(rows), REQUEST_DTYPE)
    for k, (s, e, m) in enumerate(rows):
        out[k] = (s, e, m, 0)
    return out


def step_order(max_step):
    """The steps in their tie order: 0, -1, +1, -2, +2, ..., -max_step, +max_step."""
    return [0] + [d for k in range(1, max_step + 1) for d in (-k, k)]


def check_enable(max_trajectories, max_samples):
    """Raises ValueError where dsm_heading_enable returns DSM_E_INVALID."""
    if not (1 <= max_trajectories <= MAX_CAPACITY and 1 <= max_samples <= MAX_CAPACITY):
        raise ValueError("max_trajectories or max_samples outside [1, 2^22]")


def check_request(camera, voxel, points, offsets, rotations, K, reqs, w_unknown, w_frontier, max_trajectories=None,
                  max_samples=None):
    """(points (P, 3), offsets, rotations (n_rot, 9), requests) of a valid request; ValueError where the library
    returns DSM_E_INVALID."""
    c = G.Camera(*camera)
    fin = np.isfinite
    if not (fin(c.fx) and c.fx > 0 and fin(c.fy) and c.fy > 0 and fin(c.cx) and fin(c.cy)):
        raise ValueError("fx, fy must be finite and > 0, cx, cy finite")
    if not (1 <= c.width <= 65536 and 1 <= c.height <= 65536) or c.unknown_blocks not in (0, 1):
        raise ValueError("image size or blocking rule")
    R, v = np.float64(np.float32(c.max_range)), G._v(voxel)
    if not (fin(R) and R > 0 and R <= G.MAX_RANGE_VOXELS * v):
        raise ValueError("max_range must be finite, > 0 and at most 128 voxels")
    rot = np.asarray(rotations, np.float64).reshape(-1, 9)
    if not (1 <= len(rot) <= MAX_ROTATIONS) or not fin(rot).all():
        raise ValueError("n_rot outside [1, 64] or a rotation entry not finite")
    if not (1 <= K <= MAX_K):
        raise ValueError("K outside [1, 64]")
    if not (0 <= w_unknown <= MAX_WEIGHT and 0 <= w_frontier <= MAX_WEIGHT):
        raise ValueError("a weight outside [0, 2^16]")
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    ofs = np.asarray(offsets, np.int64).reshape(-1)
    n = len(ofs) - 1
    if n < 1 or (max_trajectories is not None and n > max_trajectories):
        raise ValueError("trajectory count")
    if ofs[0] != 0 or ofs[-1] > len(pts):
        raise ValueError("offsets")
    lens = np.diff(ofs)
    if (lens < tj.MIN_POINTS).any() or (lens > tj.MAX_POINTS).any():
        raise ValueError("points per trajectory")
    pts = pts[:ofs[-1]]
    if not fin(pts).all():
        raise ValueError("non-finite control point")
    q = np.asarray(reqs, REQUEST_DTYPE).reshape(-1)
    if len(q) != n:
        raise ValueError("one request per trajectory")
    if not ((0 <= q["start"]) & (q["start"] < len(rot)) & (-1 <= q["end"]) & (q["end"] < len(rot)) & (0 <= q["max_step"]) &
            (q["max_step"] <= len(rot))).all():
        raise ValueError("start, end or max_step out of range")
    n_samples = int((K * (lens - 3) + 1).sum())
    if max_samples is not None and n_samples > max_samples:
        raise ValueError("more than max_samples samples")
    m = 2 * int(np.ceil(R / v)) + 3
    if n_samples * m ** 3 > MAX_WORK:
        raise ValueError("the work bound sum_s (2 ceil(R / v) + 3)^3 exceeds 2^31 voxel visits")
    return pts, ofs, rot, q


def sample_positions(points, offsets, K):
    """(S, 3): every trajectory's curve_samples, concatenated in trajectory order."""
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    ofs = np.asarray(offsets, np.int64).reshape(-1)
    return np.concatenate([tj.curve_samples(pts[ofs[j]:ofs[j + 1]], K) for j in range(len(ofs) - 1)])


def box_hull(t, rotations, camera, voxel, origin, shape):
    """(lo, size) of the hull of the host's gain boxes (pyoracle_gain.box) of the poses [R_r | t]; size 0 when all
    are empty."""
    lo, hi = None, None
    for R in np.asarray(rotations, np.float64).reshape(-1, 3, 3):
        a, s = G.box(np.concatenate([R, np.asarray(t, np.float64)[:, None]], axis=1).reshape(12), camera, voxel, origin, shape)
        if (s == 0).any():
            continue
        lo = a if lo is None else np.minimum(lo, a)
        hi = a + s if hi is None else np.maximum(hi, a + s)
    if lo is None:
        return np.zeros(3, np.int64), np.zeros(3, np.int64)
    return lo, hi - lo


def sample_counts(state, origin, voxel, camera, rotations, t, front=None):
    """(n_unknown (n_rot,), n_frontier (n_rot,)) int64 of a camera at t: per rotation r, the unknown and the frontier
    voxels that pass the frustum test of [R_r | t] and whose walk from t reaches them; zeros for a camera whose voxel
    lies outside the grid."""
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    rot = np.asarray(rotations, np.float64).reshape(-1, 3, 3)
    zero = np.zeros(len(rot), np.int64)
    t = np.asarray(t, np.float64)
    if not G.camera_inside(np.concatenate([np.eye(3), t[:, None]], axis=1).reshape(12), voxel, origin, (nx, ny, nz)):
        return zero, zero.copy()
    lo, size = box_hull(t, rot, camera, voxel, origin, (nx, ny, nz))
    if (size == 0).any():
        return zero, zero.copy()
    front = pyoracle_frontier.frontier_mask(st) if front is None else front
    g = np.stack(np.meshgrid(*[np.arange(lo[k], lo[k] + size[k]) for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
    c = G.centres(g, origin, voxel)
    poses = [np.concatenate([R, t[:, None]], axis=1).reshape(12) for R in rot]
    inside = np.stack([G.frustum(c, P, camera) for P in poses])      # (n_rot, n)
    anyf = inside.any(axis=0)
    g, c, inside = g[anyf], c[anyf], inside[:, anyf]
    s = G.seen(st, origin, voxel, t, c, G.Camera(*camera).unknown_blocks)
    unk = s & (st[g[:, 2], g[:, 1], g[:, 0]] == G.UNKNOWN)
    fr = s & front[g[:, 2], g[:, 1], g[:, 0]]
    return (inside & unk).sum(axis=1).astype(np.int64), (inside & fr).sum(axis=1).astype(np.int64)


def plan(score, start, end, max_step):
    """(status, rotations (S,), turns (S,), total score, sum |delta|) of one trajectory's score table (S, n_rot) int64:
    the backward pass that keeps the first best successor per (s, r) in step_order, then the forward trace from start.
    Status 1 (end unreachable): every rotation -1, every turn 0, score and steps 0."""
    score = np.asarray(score, np.int64)
    S, n_rot = score.shape
    r = np.arange(n_rot)
    ok = (r == end) if end >= 0 else np.ones(n_rot, bool)
    val = np.where(ok, score[-1], 0)
    steps = np.zeros(n_rot, np.int64)
    succ = np.zeros((S, n_rot), np.int64)
    for s in range(S - 2, -1, -1):
        b_ok, b_val, b_steps, b_d = np.zeros(n_rot, bool), np.zeros(n_rot, np.int64), np.zeros(n_rot, np.int64), np.zeros(n_rot, np.int64)
        for d in step_order(max_step):
            nxt = (r + d) % n_rot
            c_ok, c_val, c_steps = ok[nxt], val[nxt], steps[nxt] + abs(d)
            better = c_ok & (~b_ok | (c_val > b_val) | ((c_val == b_val) & (c_steps < b_steps)))
            b_ok, b_val, b_steps, b_d = b_ok | better, np.where(better, c_val, b_val), np.where(better, c_steps, b_steps), \
                np.where(better, d, b_d)
        ok, val, steps, succ[s] = b_ok, np.where(b_ok, score[s] + b_val, 0), b_steps, b_d
    if not ok[start]:
        return 1, np.full(S, -1, np.int32), np.zeros(S, np.int32), 0, 0
    rots, turns = np.zeros(S, np.int32), np.zeros(S, np.int32)
    cur, turn = start, 0
    for s in range(S):
        rots[s], turns[s] = cur, turn
        if s + 1 < S:
            turn += int(succ[s, cur])
            cur = (cur + int(succ[s, cur])) % n_rot
    return 0, rots, turns, int(val[start]), int(steps[start])


def job(state, origin, voxel, camera, rotations, K, points, offsets, reqs, w_unknown, w_frontier):
    """(info INFO_DTYPE record, records RECORD_DTYPE (n,), samples SAMPLE_DTYPE (S,), counts COUNT_DTYPE (S, n_rot)) of
    one call on the state grid [nz][ny][nx] at integer origin (x, y, z)."""
    pts, ofs, rot, q = check_request(camera, voxel, points, offsets, rotations, K, reqs, w_unknown, w_frontier)
    st = np.asarray(state, np.uint8)
    n, n_rot = len(ofs) - 1, len(rot)
    pos = sample_positions(pts, ofs, K)
    front = pyoracle_frontier.frontier_mask(st)
    counts = np.zeros((len(pos), n_rot), COUNT_DTYPE)
    outside = np.zeros(len(pos), bool)
    nz, ny, nx = st.shape
    for s, t in enumerate(pos):
        outside[s] = not G.camera_inside(np.concatenate([np.eye(3), t[:, None]], axis=1).reshape(12), voxel, origin, (nx, ny, nz))
        counts[s]["n_unknown"], counts[s]["n_frontier"] = sample_counts(st, origin, voxel, camera, rot, t, front)
    score = np.int64(w_unknown) * counts["n_unknown"].astype(np.int64) + np.int64(w_frontier) * counts["n_frontier"].astype(np.int64)
    samples = np.zeros(len(pos), SAMPLE_DTYPE)
    samples["p"] = pos
    recs = np.zeros(n, RECORD_DTYPE)
    info = np.zeros((), INFO_DTYPE)
    base = 0
    for j in range(n):
        S = K * (int(ofs[j + 1] - ofs[j]) - 3) + 1
        status, rots, turns, total, steps = plan(score[base:base + S], int(q[j]["start"]), int(q[j]["end"]), int(q[j]["max_step"]))
        samples["rotation"][base:base + S], samples["turn"][base:base + S] = rots, turns
        recs[j] = (status, S, base, int(outside[base:base + S].sum()), total, steps, 0)
        info["n_status"][status] += 1
        base += S
    info["origin"] = np.asarray(origin, np.int32)
    info["n_trajectories"], info["n_samples"], info["n_rot"] = n, len(pos), n_rot
    info["unknown_blocks"] = G.Camera(*camera).unknown_blocks
    return info, recs, samples, counts
