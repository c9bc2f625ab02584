"""Surfel pools built from a frame's seed table so that the surfel fuse and initialise (k_fuse, k_init_surfels; host model
oracle/pyoracle_fuse.py) reach every outcome, with a pair of neighbouring floats on each side of every threshold.
Shared by tests/test_fuse_model.py (the model against the reference's own fuse, on the CPU) and tests/test_gpu_fuse.py
(the kernels against the model, on the device's own seeds).

A pool is a function of the seeds, so the same builder serves the reference's seeds and the device's: each comparison
builds its pool from the seeds of the side it checks.  Each threshold is found by bisection over the float bit patterns
of one surfel field, with the model deciding the branch: the pool then holds the last float that takes one branch and
the first that takes the other.
"""
import numpy as np

import pyoracle
import pyoracle_fuse as pf
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE

F32 = np.float32
CTA = 1024  # seeds per k_init_surfels CTA


# ---- frames: (camera, frame id, depth scale); each runs with both constant sets ----
FRAMES = {
    "vga": (synth.VGA, 0, 1.0),
    "kitti": (synth.KITTI, 5, 1.0),  # 1226 wide: the device row pitch (1232) exceeds the width
    # 14 400 seeds, 15 k_init_surfels CTAs; fuse_far 60 m so that every seed, the 40 m backdrop too, can be fused
    "hd": (synth.Camera(1280, 720, 720.0, 720.0, 639.5, 359.5, 0.5, 60.0), 4, 1.0),
    "near": (synth.VGA, 0, 0.02),    # every depth under 1 m: get_weight's clamp, NaN mean depths
}
# three different VGA frames for the batch slots
BATCH_FRAMES = ("vga", "near", "vga2")
EXTRA_FRAMES = {"vga2": (synth.VGA, 2, 1.0)}
CONSTANTS = {"drive": pyoracle.CONSTANTS_DRIVE, "rgbd": pyoracle.CONSTANTS_RGBD}


def frame(name):
    cam, fid, scale = {**FRAMES, **EXTRA_FRAMES}[name]
    gray, depth = synth.make_frame(cam, fid, synth.pose_stream(fid))
    return cam, gray, (depth * F32(scale)).astype(F32)


def general_pose():
    """A rotation of 25 degrees about an oblique axis with a translation: column-major float32[16]."""
    ax = np.array([0.3, -0.8, 0.52])
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(25.0)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    T[:3, 3] = [1.5, -0.7, 3.2]
    return np.ascontiguousarray(T.T.astype(F32).reshape(16))


POSES = {"identity": synth.identity_pose(), "general": general_pose()}


# ---- float bit patterns in value order ----
def _key(x):
    i = np.asarray(x, F32).view(np.int32).astype(np.int64)
    return np.where(i >= 0, i, -(i & 0x7FFFFFFF))


def _unkey(k):
    k = np.asarray(k, np.int64)
    i = np.where(k >= 0, k, (-k) | 0x80000000).astype(np.uint32)
    return i.view(F32)


class Frame:
    """One frame's inputs to the fuse step: seeds, labels, depth, pose, constants and the reference frame index."""

    def __init__(self, cam, seeds, labels, depth, pose, constants, ref):
        self.cam, self.labels, self.depth, self.constants, self.ref = cam, labels, depth, constants, ref
        self.seeds = np.array(seeds, copy=True)
        self.seeds["fused"] = 0
        self.pose = np.asarray(pose, F32).reshape(16)
        self.ipose = pf.inverse4f(self.pose)
        self.T = self.pose.astype(np.float64).reshape(4, 4).T

    def run(self, pool, mutation=None):
        return pf.fuse(self.seeds, self.labels, self.depth, self.pose, self.ipose, self.cam, self.constants, self.ref,
                       pool, mutation)

    def outcome(self, pool):
        return self.run(pool)["outcome"]

    def surfel(self, u, v, z, n_cam, size=0.05, weight=1.0, update_times=6, last_update=None):
        """Surfels at camera depth z on the rays through pixels (u, v), camera-frame normals n_cam, sent to world."""
        u, v, z = (np.atleast_1d(np.asarray(a, np.float64)) for a in (u, v, z))
        c = self.cam
        pc = np.stack([(u - c.cx) / c.fx * z, (v - c.cy) / c.fy * z, z, np.ones_like(z)], -1)
        pw = pc @ self.T.T
        nw = np.asarray(n_cam, np.float64).reshape(-1, 3) @ self.T[:3, :3].T
        s = np.zeros(len(z), SURFEL_DTYPE)
        s["px"], s["py"], s["pz"] = pw[:, 0], pw[:, 1], pw[:, 2]
        s["nx"], s["ny"], s["nz"] = nw[:, 0], nw[:, 1], nw[:, 2]
        s["size"], s["weight"], s["update_times"] = size, weight, update_times
        s["last_update"] = self.ref - 1 if last_update is None else last_update
        s["color"] = 77.25
        return s

    def seed_normal(self, s):
        sd = self.seeds[s]
        return np.stack([sd["norm_x"], sd["norm_y"], sd["norm_z"]], -1).astype(np.float64)

    def usable(self):
        """Seeds a surfel can fuse into: finite positive mean depth inside the fuse range, a normal, view_cos >= 0.1."""
        sd = self.seeds
        nz = ~((sd["norm_x"] == 0) & (sd["norm_y"] == 0) & (sd["norm_z"] == 0))
        md = sd["mean_depth"]
        with np.errstate(invalid="ignore"):
            return np.nonzero(nz & np.isfinite(md) & (md > self.cam.near * 1.01) & (md < self.cam.far * 0.99)
                              & (sd["view_cos"].astype(np.float64) >= 0.1)
                              & np.isfinite(sd["norm_x"]) & np.isfinite(sd["view_cos"]))[0]

    def fusers(self, want):
        """For each seed of `want`, a surfel that fuses into it (size 1: the seed's size is kept unless smaller);
        seeds for which no pixel works are left out.  Returns (surfels, seeds they fuse into)."""
        H, W = self.labels.shape
        flat = self.labels.reshape(-1)
        order = np.argsort(flat, kind="stable")
        starts = np.searchsorted(flat[order], np.arange(len(self.seeds) + 1))
        sd = self.seeds
        got_s, got_i = [], []
        want = np.asarray(want)
        cx = np.rint(sd["x"][want]).astype(int)
        cy = np.rint(sd["y"][want]).astype(int)
        # candidate pixels: the seed's centre first, then its pixels in raster order
        cands = []
        for k, s in enumerate(want):
            px = order[starts[s]:starts[s + 1]]
            pu, pv = px % W, px // W
            d = (pu - cx[k]) ** 2 + (pv - cy[k]) ** 2
            pick = px[np.argsort(d, kind="stable")][:24]
            cands.append(pick)
        for r in range(24):
            idx = [k for k in range(len(want)) if len(cands[k]) > r]
            if not idx:
                break
            pix = np.array([cands[k][r] for k in idx])
            ss = want[idx]
            surf = self.surfel(pix % W, pix // W, sd["mean_depth"][ss], self.seed_normal(ss), size=1.0)
            res = self.run(surf)
            ok = (res["outcome"] >= pf.FUSED_SHRUNK) & (res["sp"] == ss)
            for j in np.nonzero(ok)[0]:
                got_s.append(surf[j])
                got_i.append(ss[j])
            done = set(ss[ok].tolist())
            for k in idx:
                if want[k] in done:
                    cands[k] = []
        return np.array(got_s, SURFEL_DTYPE), np.array(got_i, np.int64)

    def bisect(self, base, field, lo, hi, want_lo, want_hi):
        """For each base surfel: the neighbouring floats t0 < t1 of `field` between lo and hi where the branch changes
        from want_lo (at t0) to want_hi (at t1).  want_* = None: any other branch than the other side's.  Returns the
        two surfels of every probe whose end points took the wanted branches (and whose last pair still does)."""
        base = np.array(base, copy=True)
        klo, khi = _key(lo), _key(hi)

        def at(keys):
            s = base.copy()
            s[field] = _unkey(keys)
            return s, self.outcome(s)

        def good(o_lo, o_hi):
            return (o_lo != o_hi) & ((o_lo == want_lo) if want_lo is not None else True) & \
                ((o_hi == want_hi) if want_hi is not None else True)

        _, o_lo = at(klo)
        _, o_hi = at(khi)
        keep = good(o_lo, o_hi)
        klo, khi, o_lo, o_hi, base = klo[keep], khi[keep], o_lo[keep], o_hi[keep], base[keep]
        while len(base) and (khi - klo > 1).any():
            mid = (klo + khi) // 2
            _, o = at(mid)
            left = o == o_lo  # still the low side's branch
            klo = np.where(left, mid, klo)
            khi = np.where(left, khi, mid)
        a, oa = at(klo)
        b, ob = at(khi)
        ok = good(oa, ob)
        return a[ok], b[ok]


def _spread(idx, k):
    """k indices spread evenly over idx."""
    idx = np.asarray(idx)
    if len(idx) <= k:
        return idx
    return idx[np.linspace(0, len(idx) - 1, k).round().astype(int)]


def build(fr, per_threshold=4, natural=160):
    """The crafted pool of one frame: returns (pool, probes) where probes maps a threshold name to a list of
    (i0, i1) pool index pairs, the last float of one branch and the first of the other."""
    cam, sd = fr.cam, fr.seeds
    H, W = fr.labels.shape
    parts, probes = [], {}
    n0 = [0]

    def add(s):
        parts.append(s)
        i = n0[0]
        n0[0] += len(s)
        return i

    def add_pairs(name, a, b):
        i = add(a)
        j = add(b)
        probes.setdefault(name, []).extend((i + k, j + k) for k in range(len(a)))

    use = fr.usable()
    md = sd["mean_depth"].astype(np.float64)

    # fusing surfels into a spread of seeds, sizes on both sides of the seed's new size
    nat, nat_s = fr.fusers(_spread(use, natural))
    nat["size"] = np.where(np.arange(len(nat)) % 2 == 0, F32(1.0), F32(1e-3))
    add(nat)
    base = nat[:1]

    # stability: ref - last_update at 5 and 6, update_times at 4 and 5; update_times == 0
    for age in (5, 6):
        for times in (4, 5):
            s = base.copy()
            s["last_update"], s["update_times"] = fr.ref - age, times
            add(s)
    for age in (0, 9):
        s = base.copy()
        s["last_update"], s["update_times"] = fr.ref - age, 0
        add(s)

    # positions off the image or beyond the int range, NaN / infinite positions, a NaN normal
    zc = float(md[nat_s[0]])
    odd = fr.surfel([-1e12, 3e12, cam.cx, cam.cx, 4e9, -5e9], [cam.cy, cam.cy, 1e13, -1e13, cam.cy, cam.cy], [zc] * 6,
                    [[0, 0, -1]] * 6)
    add(odd)
    for f, v in (("px", np.nan), ("py", np.nan), ("pz", np.nan), ("px", np.inf), ("pz", np.inf), ("pz", -np.inf),
                 ("py", -np.inf)):
        s = base.copy()
        s[f] = v
        add(s)
    s = base.copy()
    s["nx"] = np.nan
    add(s)

    # a surfel on a zero-normal seed and on a low-view_cos seed
    zero = np.nonzero((sd["norm_x"] == 0) & (sd["norm_y"] == 0) & (sd["norm_z"] == 0) & (sd["mean_depth"] > 0))[0]
    with np.errstate(invalid="ignore"):
        low = np.nonzero(~((sd["norm_x"] == 0) & (sd["norm_y"] == 0) & (sd["norm_z"] == 0))
                         & (sd["view_cos"].astype(np.float64) < 0.1) & np.isfinite(sd["mean_depth"]))[0]
    for group in (_spread(zero, 4), low):
        for s in group:
            u, v = int(round(float(sd["x"][s]))), int(round(float(sd["y"][s])))
            z = float(fr.depth[v, u]) if fr.depth[v, u] > 0 else float(md[s])
            add(fr.surfel(u, v, max(z, cam.near * 1.5), [[0, 0, -1]]))

    pick = _spread(np.arange(len(nat)), per_threshold)
    ps = nat_s[pick]
    ray_u = np.rint(sd["x"][ps]).astype(int)
    ray_v = np.rint(sd["y"][ps]).astype(int)
    nrm = fr.seed_normal(ps)

    def along_z(z_lo, z_hi, uu, vv, nn):
        a = fr.surfel(uu, vv, z_lo, nn)
        b = fr.surfel(uu, vv, z_hi, nn)
        f = _z_field(fr)
        return a, f, a[f], b[f]

    # near / far
    for name, zt, wl, wh in (("near", cam.near, pf.NEAR, None), ("far", cam.far, None, pf.FAR)):
        zt = np.full(len(ps), zt)
        a, f, lo, hi = along_z(zt * (1 - 1e-3), zt * (1 + 1e-3), ray_u, ray_v, nrm)
        add_pairs(name, *fr.bisect(a, f, lo, hi, wl, wh))

    # occlusion: depth - 1.0 at the pixel
    dd = fr.depth[ray_v, ray_u].astype(np.float64) - 1.0
    okd = (dd > cam.near * 1.1) & (dd < cam.far * 0.9)
    if okd.any():
        a, f, lo, hi = along_z(dd[okd] * (1 - 1e-4), dd[okd] * (1 + 1e-4), ray_u[okd], ray_v[okd], nrm[okd])
        add_pairs("occlusion", *fr.bisect(a, f, lo, hi, pf.OCCLUDING, None))

    # mean_depth -+ tol, on both sides of the min_tolerate_diff clamp
    _, baseline, derr, mintol = fr.constants
    cf = float(pf.camera_f(cam))
    tol_of = lambda z: np.maximum(z * z / (baseline * cf) * derr, mintol)
    cand = fr.usable()
    clamp = tol_of(md[cand]) <= mintol
    for side, sel in (("clamped", cand[clamp]), ("computed", cand[~clamp])):
        sel = _spread(sel, per_threshold)
        if not len(sel):
            continue
        su, sv = np.rint(sd["x"][sel]).astype(int), np.rint(sd["y"][sel]).astype(int)
        keep = fr.labels[sv, su] == sel
        sel, su, sv = sel[keep], su[keep], sv[keep]
        for name, sign, wl, wh in (("too_near", -1, pf.TOO_NEAR, None), ("too_far", 1, None, pf.TOO_FAR)):
            # tol is taken at the surfel's own depth: the threshold is the fixed point z = mean_depth + sign * tol(z)
            thr = md[sel].copy()
            with np.errstate(all="ignore"):
                for _ in range(60):
                    thr = md[sel] + sign * tol_of(thr)
                inside = ((np.abs(thr - md[sel] - sign * tol_of(thr)) < 1e-9 * thr) & (thr > cam.near * 1.1)
                          & (thr < cam.far * 0.99) & (fr.depth[sv, su] - 1.0 < thr * 0.999))  # not occluding
            if not inside.any():
                continue
            t = thr[inside]
            w = 1e-2 * tol_of(t) / t
            a, f, lo, hi = along_z(t * (1 - w), t * (1 + w), su[inside], sv[inside], fr.seed_normal(sel[inside]))
            add_pairs(f"{name} ({side})", *fr.bisect(a, f, lo, hi, wl, wh))

    # ndc against 0.1: vary the world normal component that moves ndc most
    n_s = nrm
    q = np.cross(n_s, np.where(np.abs(n_s[:, :1]) < 0.9, [[1.0, 0, 0]], [[0, 1.0, 0]]))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    a = fr.surfel(ray_u, ray_v, md[ps], q - 0.2 * n_s)
    b = fr.surfel(ray_u, ray_v, md[ps], q + 0.5 * n_s)
    Rn = n_s @ fr.T[:3, :3].T
    k = np.argmax(np.abs(Rn), axis=1)
    for f in ("nx", "ny", "nz"):
        sel = k == "xyz".index(f[1])
        if sel.any():
            a2 = a[sel].copy()
            lo, hi = a[f][sel], b[f][sel]
            sw = lo > hi
            lo2, hi2 = np.where(sw, hi, lo), np.where(sw, lo, hi)
            wl = np.where(sw, None, pf.NORMAL_MISMATCH)
            for flip in (False, True):
                m = sw == flip
                if m.any():
                    add_pairs("ndc", *fr.bisect(a2[m], f, lo2[m], hi2[m], None if flip else pf.NORMAL_MISMATCH,
                                                pf.NORMAL_MISMATCH if flip else None))

    # pixel rounding at the image borders: ui in {0, 1} and {W-2, W-1}, vi likewise
    rows = np.linspace(H * 0.3, H * 0.7, per_threshold).astype(int)
    cols = np.linspace(W * 0.3, W * 0.7, per_threshold).astype(int)
    for name, axis, at_lo, at_hi, wl, wh in (("u 0|1", 0, 0, 1, pf.BORDER, None), ("u W-2|W-1", 0, W - 2, W - 1, None, pf.BORDER),
                                             ("v 0|1", 1, 0, 1, pf.BORDER, None), ("v H-2|H-1", 1, H - 2, H - 1, None, pf.BORDER)):
        other = rows if axis == 0 else cols
        uu_lo, vv_lo = (np.full_like(other, at_lo), other) if axis == 0 else (other, np.full_like(other, at_lo))
        uu_hi, vv_hi = (np.full_like(other, at_hi), other) if axis == 0 else (other, np.full_like(other, at_hi))
        z = fr.depth[vv_hi.clip(1, H - 2), uu_hi.clip(1, W - 2)].astype(np.float64)
        z = np.where((z > cam.near * 1.2) & (z < cam.far * 0.9), z, 5.0)
        lo_s = fr.surfel(uu_lo, vv_lo, z, [[0, 0, -1]] * len(z))
        hi_s = fr.surfel(uu_hi, vv_hi, z, [[0, 0, -1]] * len(z))
        f = _uv_field(fr, axis)
        lo, hi = lo_s[f], hi_s[f]
        sw = lo > hi
        for flip in (False, True):
            m = sw == flip
            if m.any():
                l2, h2 = (hi[m], lo[m]) if flip else (lo[m], hi[m])
                add_pairs(name, *fr.bisect(lo_s[m], f, l2, h2, wh if flip else wl, wl if flip else wh))

    # the size update: new_size against size
    res = fr.run(nat[pick])
    fz = res["outcome"] >= pf.FUSED_SHRUNK
    if fz.any():
        s = nat[pick][fz]
        ns = pf.new_size(sd["size"][res["sp"][fz]], sd["mean_depth"][res["sp"][fz]], sd["view_cos"][res["sp"][fz]],
                         pf.camera_f(cam))
        add_pairs("size", *fr.bisect(s, "size", (ns * F32(0.5)).astype(F32), (ns * F32(2)).astype(F32),
                                     pf.FUSED_KEPT, pf.FUSED_SHRUNK))
    return np.concatenate(parts), probes


def _z_field(fr):
    """The world position field that moves the camera-frame z most (row 2 of the inverse pose)."""
    return ("px", "py", "pz")[int(np.argmax(np.abs(fr.ipose.reshape(4, 4).T[2, :3])))]


def _uv_field(fr, axis):
    """The world position field that moves camera-frame x (axis 0) or y (axis 1) most."""
    return ("px", "py", "pz")[int(np.argmax(np.abs(fr.ipose.reshape(4, 4).T[axis, :3])))]


# ---- k_init_surfels: emit patterns around the 1024-seed CTA boundaries ----
INIT_PATTERNS = ("none_before", "boundary_pair", "alternating", "cta_full")


def boundary_pair(fr):
    """The two seeds around the first CTA boundary that can both emit: 1023 and 1024 when they can."""
    cap = np.zeros(len(fr.seeds), bool)
    cap[fr.usable()] = True
    b = next(b for b in range(CTA, len(fr.seeds), CTA) if cap[b - 1] and cap[b])
    return b - 1, b


def init_pool(fr, pattern):
    """Fusing surfels that mark seeds fused so that the emitting seeds follow `pattern`:
    none_before     every seed of the first CTA fused: the second CTA starts with no emission before it;
    boundary_pair   every seed fused but boundary_pair's two: the only emitters straddle a CTA boundary;
    alternating     every odd seed fused: emitters alternate;
    cta_full        every seed of the sixth CTA fused."""
    S = len(fr.seeds)
    cap = np.zeros(S, bool)
    cap[fr.usable()] = True
    idx = np.arange(S)
    pair = boundary_pair(fr) if pattern == "boundary_pair" else (-1, -1)
    mark = {"none_before": idx < CTA, "boundary_pair": (idx != pair[0]) & (idx != pair[1]),
            "alternating": idx % 2 == 1, "cta_full": (idx >= 5 * CTA) & (idx < 6 * CTA)}[pattern]
    pool, _ = fr.fusers(np.nonzero(mark & cap)[0])
    return pool


def pad(pool, n, seed=0):
    """The pool grown to n surfels with dead ones (update_times 0) at the end: sets the slice lengths of a batch."""
    extra = n - len(pool)
    assert extra >= 0
    fill = np.zeros(extra, SURFEL_DTYPE)
    rng = np.random.RandomState(seed)
    fill["px"], fill["py"], fill["pz"] = rng.uniform(-5, 5, (3, extra))
    fill["nz"] = 1
    fill["last_update"] = 0
    return np.concatenate([pool, fill])


def margin(fr, pool):
    """Per surfel, the smallest relative distance of the seed-dependent decisions the model took for it from their
    thresholds (mean_depth -+ tol, ndc, the seed's view_cos, new_size against size); inf when it took none.  The
    other decisions depend only on the pose, the depth image and the surfel, which both sides compute alike."""
    r = fr.run(pool)
    o = r["outcome"]
    z, md, tol, ndc = (r[k].astype(np.float64) for k in ("z", "md", "tol", "ndc"))
    vc = fr.seeds["view_cos"][r["sp"]].astype(np.float64)
    m = np.full(len(pool), np.inf)
    with np.errstate(all="ignore"):
        reach_vc = o >= pf.LOW_VIEW_COS
        m = np.where(reach_vc, np.minimum(m, np.abs(vc - 0.1)), m)
        reach_tol = o >= pf.TOO_NEAR
        sc = np.maximum(np.abs(md), 1.0)
        m = np.where(reach_tol, np.minimum(m, np.abs(z - (md - tol)) / sc), m)
        m = np.where(o >= pf.TOO_FAR, np.minimum(m, np.abs(z - (md + tol)) / sc), m)
        m = np.where(o >= pf.NORMAL_MISMATCH, np.minimum(m, np.abs(ndc - 0.1)), m)
        fz = o >= pf.FUSED_SHRUNK
        sp = r["sp"]
        ns = pf.new_size(fr.seeds["size"][sp], fr.seeds["mean_depth"][sp], fr.seeds["view_cos"][sp], pf.camera_f(fr.cam))
        rel = np.abs(ns.astype(np.float64) - pool["size"]) / np.maximum(np.abs(pool["size"].astype(np.float64)), 1e-30)
        m = np.where(fz, np.minimum(m, rel), m)
    return np.where(np.isnan(m), 0.0, m)
