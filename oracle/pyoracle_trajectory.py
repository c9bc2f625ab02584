"""The trajectory job of dsm_trajectory_* (DESIGN.md §8.17, include/dsm.h) restated in numpy: L-BFGS with Armijo
backtracking over the free control points of uniform cubic B-splines against the signed grid of
oracle/pyoracle_field_signed, and the final clearance check of the optimised curves.

Every step is float64 with one rounding per operation, as the library computes it (it is built with -fmad=false and
uses explicit _rn intrinsics), except the field samples, which are the float32 signed point queries widened to float64.
Every sum over points is the library's warp reduction restated with ordered adds (reduce()), never np.sum, so the
restatement is bit for bit."""
import numpy as np

import pyoracle_field_signed

MAX_POINTS = 256            # DSM_TRAJECTORY_MAX_POINTS: control points of one trajectory
MIN_POINTS = 7
MAX_MEMORY = 16
MAX_ITER = 1024
MAX_LS = 32
MAX_K = 64
MAX_WORK = 1 << 32          # sum of N_j * max_iter * (max_ls + 1)
MAX_SAMPLES = 1 << 26       # final samples of one call
C1 = 1e-4
FIXED = 3                   # fixed control points at each end

RECORD_DTYPE = np.dtype([("status", "<i4"), ("iterations", "<i4"), ("evaluations", "<i4"), ("n_free_outside", "<i4"),
                         ("cost_start", "<f8"), ("cost", "<f8"), ("smoothness", "<f8"), ("clearance", "<f8"),
                         ("feasibility", "<f8"), ("max_v", "<f8"), ("max_a", "<f8"), ("min_dist", "<f4"), ("argmin", "<i4"),
                         ("first_hit", "<i4"), ("n_outside", "<i4"), ("reserved", "<i4", 2)])
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_trajectories", "<i4"), ("n_points", "<i4"), ("n_status", "<i4", 4),
                       ("reserved", "<i4", 7)])
PARAM_NAMES = ("w_smooth", "w_clear", "w_feas", "margin", "v_max", "a_max", "g_tol", "max_iter", "memory", "max_ls",
               "samples", "radius")


def params(w_smooth=1.0, w_clear=10.0, w_feas=1.0, margin=0.5, v_max=2.0, a_max=2.0, g_tol=1e-6, max_iter=100, memory=8,
           max_ls=16, samples=8, radius=0.3):
    """The parameters of one call as a dict (the fields of dsm_trajectory_params_t)."""
    return dict(w_smooth=float(w_smooth), w_clear=float(w_clear), w_feas=float(w_feas), margin=float(margin),
                v_max=float(v_max), a_max=float(a_max), g_tol=float(g_tol), max_iter=int(max_iter), memory=int(memory),
                max_ls=int(max_ls), samples=int(samples), radius=float(np.float32(radius)))


def reduce(v):
    """The library's sum of the values v[k], k = 0 .. n-1: lane l = k mod 32 adds its values in ascending k to 0.0,
    then a butterfly (each lane adds the lane l ^ m for m = 16, 8, 4, 2, 1) leaves every lane with the same bits."""
    v = np.asarray(v, np.float64).reshape(-1)
    rows = -(-len(v) // 32)
    pad = np.zeros(rows * 32, np.float64)   # lanes past the end add nothing: +0.0 leaves a sum that is never -0.0
    pad[:len(v)] = v
    acc = np.zeros(32, np.float64)
    for r in range(rows):
        acc = acc + pad[32 * r:32 * r + 32]
    lane = np.arange(32)
    for m in (16, 8, 4, 2, 1):
        acc = acc + acc[lane ^ m]
    return acc[0]


def dot(a, b):
    """gᵀd-style product of two (M, 3) arrays over the free points: ((ax bx + ay by) + az bz) per point, reduce()d."""
    return reduce((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2])


def grid_sampler(sdist, origin, voxel):
    """The sampler of the signed grid: points (n, 3) -> (inside, d, grad (n, 3)), the float32 signed point query widened
    to float64."""
    def sampler(p):
        s = pyoracle_field_signed.sample(sdist, origin, voxel, p)
        inside = ~np.isnan(s["dist"])
        g = np.stack([s["gx"], s["gy"], s["gz"]], 1).astype(np.float64)
        return inside, s["dist"].astype(np.float64), g
    return sampler


def jerk(Q):
    """(N - 3, 3): (Q[i+3] - Q[i]) + 3 (Q[i+1] - Q[i+2])."""
    return (Q[3:] - Q[:-3]) + 3.0 * (Q[1:-2] - Q[2:-1])


def _pen(t):
    return np.where(t > 0.0, t * t, 0.0)


def evaluate(Q, dt, p, sampler):
    """(J, (J_s, J_c, J_f), g (M, 3), free points outside) at control points Q (N, 3); M = N - 6 free points."""
    N = len(Q)
    dt2 = dt * dt
    v2, a2 = p["v_max"] * p["v_max"], p["a_max"] * p["a_max"]
    j = jerk(Q)
    Js = reduce((j[:, 0] * j[:, 0] + j[:, 1] * j[:, 1]) + j[:, 2] * j[:, 2])
    V = (Q[1:] - Q[:-1]) / dt
    A = ((Q[2:] - Q[1:-1]) - (Q[1:-1] - Q[:-2])) / dt2
    tv, ta = V * V - v2, A * A - a2
    fv, fa = _pen(tv), _pen(ta)
    Jf = reduce((fv[:, 0] + fv[:, 1]) + fv[:, 2]) + reduce((fa[:, 0] + fa[:, 1]) + fa[:, 2])
    free = np.arange(FIXED, N - FIXED)
    inside, d, gd = sampler(Q[free])
    with np.errstate(invalid="ignore"):
        e = p["margin"] - d
        hit = inside & (e > 0.0)   # outside (NaN) and +inf (no site) contribute nothing
        Jc = reduce(np.where(hit, e * e, 0.0))
        gc = np.where(hit[:, None], (-2.0 * e)[:, None] * gd, 0.0)
    # smoothness: the terms i-3, i-2, i-1, i that hold Q_i, at coefficients 1, -3, 3, -1, times 2
    i = free
    gs = 2.0 * (((j[i - 3] - 3.0 * j[i - 2]) + 3.0 * j[i - 1]) - j[i])
    dv = np.where(tv > 0.0, (4.0 * tv) * V, 0.0)
    da = np.where(ta > 0.0, (4.0 * ta) * A, 0.0)
    gf = (dv[i - 1] - dv[i]) / dt + ((da[i - 2] - 2.0 * da[i - 1]) + da[i]) / dt2
    g = (p["w_smooth"] * gs + p["w_clear"] * gc) + p["w_feas"] * gf
    J = (p["w_smooth"] * Js + p["w_clear"] * Jc) + p["w_feas"] * Jf
    return J, (Js, Jc, Jf), g, int((~inside).sum())


def basis(u):
    """The uniform cubic B-spline basis at u (fp64, the stated order)."""
    u = np.float64(u)
    u2 = u * u
    u3 = u2 * u
    w = 1.0 - u
    b0 = ((w * w) * w) / 6.0
    b1 = ((3.0 * u3 - 6.0 * u2) + 4.0) / 6.0
    b2 = (((3.0 * u2 - 3.0 * u3) + 3.0 * u) + 1.0) / 6.0
    b3 = u3 / 6.0
    return b0, b1, b2, b3


def curve_samples(Q, K):
    """(S, 3): segments m = 0 .. N-4 at u = s / K, s < K, then the end point (segment N-4 at u = 1)."""
    N = len(Q)
    s = np.arange((N - 3) * K + 1)
    m = np.minimum(s // K, N - 4)
    u = (s - m * K).astype(np.float64) / np.float64(K)
    b0, b1, b2, b3 = basis(u)
    return ((b0[:, None] * Q[m] + b1[:, None] * Q[m + 1]) + b2[:, None] * Q[m + 2]) + b3[:, None] * Q[m + 3]


def final_check(Q, dt, K, radius, sdist, origin, voxel):
    """(min_dist, argmin, first_hit, n_outside, max_v, max_a) of control points Q: signed distance samples of the curve."""
    pts = curve_samples(Q, K)
    d = pyoracle_field_signed.sample(sdist, origin, voxel, pts)["dist"]
    inside = ~np.isnan(d)
    if inside.any():
        mind = np.float32(d[inside].min())
        arg = int(np.flatnonzero(inside & (d == mind))[0])
    else:
        mind, arg = np.float32(np.inf), -1
    hits = np.flatnonzero(inside & (d < np.float32(radius)))
    V = np.abs((Q[1:] - Q[:-1]) / dt)
    A = np.abs(((Q[2:] - Q[1:-1]) - (Q[1:-1] - Q[:-2])) / (dt * dt))
    return mind, arg, int(hits[0]) if len(hits) else -1, int((~inside).sum()), float(np.fmax.reduce(V.reshape(-1))), \
        float(np.fmax.reduce(A.reshape(-1)))


def optimise(Q0, dt, p, sampler, voxel):
    """(Q, record fields) of one trajectory: the optimiser of include/dsm.h literally."""
    Q = np.array(Q0, np.float64).reshape(-1, 3)
    N = len(Q)
    rec = dict(status=1, iterations=0, evaluations=1)
    J, terms, g, nout = evaluate(Q, dt, p, sampler)
    rec["cost_start"] = J
    mem = p["memory"]
    S, Y, SY, YY = [None] * mem, [None] * mem, [0.0] * mem, [0.0] * mem
    h, head = 0, mem - 1
    v = np.float64(np.float32(voxel))
    while True:
        if np.fmax.reduce(np.abs(g).reshape(-1), initial=0.0) <= p["g_tol"]:
            rec["status"] = 0
            break
        if rec["iterations"] == p["max_iter"]:
            rec["status"] = 1
            break
        steep = h == 0
        if not steep:
            q = g.copy()
            alpha = [0.0] * mem
            for t in range(h):                                # newest to oldest
                k = (head - t) % mem
                alpha[k] = (1.0 / SY[k]) * dot(S[k], q)
                q = q - alpha[k] * Y[k]
            k = head
            r = (SY[k] / YY[k]) * q
            for t in range(h - 1, -1, -1):                    # oldest to newest
                k = (head - t) % mem
                beta = (1.0 / SY[k]) * dot(Y[k], r)
                r = r + S[k] * (alpha[k] - beta)
            d = -r
            gd = dot(g, d)
            if not gd < 0.0:
                h, steep = 0, True
        if steep:
            d = -g
            gd = dot(g, d)
            step = v / np.sqrt(dot(g, g))
        else:
            step = 1.0
        accepted = False
        for _ in range(p["max_ls"]):
            Qt = Q.copy()
            Qt[FIXED:N - FIXED] = Q[FIXED:N - FIXED] + step * d
            Jt, tt, gt, nt = evaluate(Qt, dt, p, sampler)
            rec["evaluations"] += 1
            if Jt <= J + (C1 * step) * gd:
                accepted = True
                break
            step = step * 0.5
        if not accepted:
            rec["status"] = 2
            break
        s = Qt[FIXED:N - FIXED] - Q[FIXED:N - FIXED]
        y = gt - g
        sy = dot(s, y)
        if sy > 0.0:
            head = (head + 1) % mem
            S[head], Y[head], SY[head], YY[head] = s, y, sy, dot(y, y)
            h = min(h + 1, mem)
        Q, J, terms, g, nout = Qt, Jt, tt, gt, nt
        rec["iterations"] += 1
    rec.update(cost=J, smoothness=terms[0], clearance=terms[1], feasibility=terms[2], n_free_outside=nout)
    return Q, rec


def check_request(points, offsets, dt, p, n_max=None, points_max=None, memory_max=MAX_MEMORY):
    """(points (P, 3), offsets, dt) of a valid request; ValueError where the library returns DSM_E_INVALID."""
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    ofs = np.asarray(offsets, np.int64).reshape(-1)
    dt = np.asarray(dt, np.float64).reshape(-1)
    n = len(ofs) - 1
    if n < 1 or (n_max is not None and n > n_max) or len(dt) != n:
        raise ValueError("trajectory count")
    if ofs[0] != 0 or ofs[-1] > len(pts) or (points_max is not None and ofs[-1] > points_max):
        raise ValueError("offsets")
    lens = np.diff(ofs)
    if (lens < MIN_POINTS).any() or (lens > MAX_POINTS).any():
        raise ValueError("points per trajectory")
    pts = pts[:ofs[-1]]
    if not np.isfinite(pts).all() or not (np.isfinite(dt) & (dt > 0)).all():
        raise ValueError("non-finite control point or dt")
    for name in ("w_smooth", "w_clear", "w_feas", "margin", "v_max", "a_max", "g_tol"):
        if not (np.isfinite(p[name]) and p[name] >= 0):
            raise ValueError(name)
    if not (0 <= p["max_iter"] <= MAX_ITER and 1 <= p["memory"] <= memory_max and 1 <= p["max_ls"] <= MAX_LS
            and 1 <= p["samples"] <= MAX_K and np.isfinite(p["radius"]) and p["radius"] >= 0):
        raise ValueError("parameters out of range")
    if int(ofs[-1]) * p["max_iter"] * (p["max_ls"] + 1) > MAX_WORK:
        raise ValueError("more than 2^32 field samples of optimisation")
    if int(((lens - 3) * p["samples"] + 1).sum()) > MAX_SAMPLES:
        raise ValueError("more than 2^26 final samples")
    return pts, ofs, dt


def job(points, offsets, dt, p, sdist, origin, voxel, sampler=None):
    """(points (P, 3), RECORD_DTYPE (n,), INFO_DTYPE record) of one call on the signed grid sdist (float32 [nz][ny][nx],
    origin in voxels, edge voxel); sampler (optional) replaces the grid's samples during the optimisation."""
    pts, ofs, dts = check_request(points, offsets, dt, p)
    sdist = np.asarray(sdist, np.float32)
    n = len(ofs) - 1
    out = pts.copy()
    recs = np.zeros(n, RECORD_DTYPE)
    info = np.zeros(1, INFO_DTYPE)[0]
    info["origin"] = np.asarray(origin, np.int32)
    info["n_trajectories"], info["n_points"] = n, ofs[-1]
    no_f = bool(np.isneginf(sdist).all())
    if sampler is None:
        sampler = grid_sampler(sdist, origin, voxel)
    for t in range(n):
        Q0 = pts[ofs[t]:ofs[t + 1]]
        if no_f:
            Q, rec = Q0.copy(), dict(status=3, iterations=0, evaluations=0, n_free_outside=0, cost_start=0.0, cost=0.0,
                                     smoothness=0.0, clearance=0.0, feasibility=0.0)
        else:
            Q, rec = optimise(Q0, dts[t], p, sampler, voxel)
        out[ofs[t]:ofs[t + 1]] = Q
        mind, arg, hit, nout, mv, ma = final_check(Q, dts[t], p["samples"], p["radius"], sdist, origin, voxel)
        rec.update(min_dist=mind, argmin=arg, first_hit=hit, n_outside=nout, max_v=mv, max_a=ma)
        for k, val in rec.items():
            recs[t][k] = val
        info["n_status"][rec["status"]] += 1
    return out, recs, info

