"""Shared comparison helpers for the parity tests (tolerances from BASELINE.json north_star /
SURVEY.md §7 H5: labels and the clustering state bit-exact, surfel geometry within 1e-4 using
norm-based metrics, integer fields exact, NaN == NaN), the golden vectors, and the drives of the reference's SurfelMap."""
import os
import zlib

import numpy as np
import pytest

import pyoracle
import pyoracle_clouds
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE

TOL = 1e-4
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CAM = synth.Camera(320, 240, 262.5, 262.5, 159.5, 119.5, 0.5, 30.0)  # quarter-VGA keeps the CPU suite short
needs_refmap_clouds = pytest.mark.skipif(not pyoracle_clouds.have_refmap_clouds(),
                                         reason="oracle/_ref/libdsm_refmap_clouds.so not built (needs the reference sources)")


def bits_equal_nan(a, b):
    """bitwise equality for float arrays except that any NaN equals any NaN."""
    a = np.asarray(a)
    b = np.asarray(b)
    both_nan = np.isnan(a) & np.isnan(b)
    return (a.view(np.uint32) == b.view(np.uint32)) | both_nan


def oracle_for(cam):
    """The parity oracle: the serialised build of the reference's own source when its prebuilt
    library is present (it travels to the GPU box inside oracle/_ref/), else the restatement
    (which test_oracle.py pins byte-for-byte to it)."""
    import pyoracle
    if pyoracle.have_reference():
        return pyoracle.RefSerial(cam)
    return pyoracle.Restatement(cam)


def check_surfels(got, want, what="surfels", tol=TOL):
    assert len(got) == len(want), f"{what}: count {len(got)} != {len(want)}"
    if len(got) == 0:
        return
    for f in ("update_times", "last_update"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, f"{what}: {f} differs at {bad[:8]} got {got[f][bad[:8]]} want {want[f][bad[:8]]}"
    pg = np.stack([got["px"], got["py"], got["pz"]], -1).astype(np.float64)
    pw = np.stack([want["px"], want["py"], want["pz"]], -1).astype(np.float64)
    ng = np.stack([got["nx"], got["ny"], got["nz"]], -1).astype(np.float64)
    nw = np.stack([want["nx"], want["ny"], want["nz"]], -1).astype(np.float64)
    nan_w = np.isnan(pw).any(1) | np.isnan(nw).any(1)
    nan_g = np.isnan(pg).any(1) | np.isnan(ng).any(1)
    assert (nan_w == nan_g).all(), f"{what}: NaN pattern differs"
    ok = ~nan_w
    pe = np.linalg.norm(pg[ok] - pw[ok], axis=1) / np.maximum(np.linalg.norm(pw[ok], axis=1), 1e-12)
    ne = np.linalg.norm(ng[ok] - nw[ok], axis=1)
    assert pe.size == 0 or pe.max() <= tol, f"{what}: position error {pe.max():.3e} > {tol}"
    assert ne.size == 0 or ne.max() <= tol, f"{what}: normal error {ne.max():.3e} > {tol}"
    for f in ("size", "weight"):
        g = got[f][ok].astype(np.float64)
        w = want[f][ok].astype(np.float64)
        fin = np.isfinite(w)
        assert (np.isfinite(g) == fin).all(), f"{what}: {f} finiteness differs"
        err = np.abs(g[fin] - w[fin]) / np.maximum(np.abs(w[fin]), 1e-12)
        assert err.size == 0 or err.max() <= tol, f"{what}: {f} error {err.max():.3e} > {tol}"
    assert bits_equal_nan(got["color"], want["color"]).all(), f"{what}: color differs"


def check_seeds(got, want, tol=TOL, cluster_exact=True):
    """Clustering state (x, y, mean_intensity, stable, and mean_depth where the plane fit rejected the seed) must be
    bit-exact; plane-fit outputs within tol."""
    assert len(got) == len(want)
    if cluster_exact:
        for f in ("x", "y", "mean_intensity"):
            bad = np.nonzero(~bits_equal_nan(got[f], want[f]))[0]
            assert len(bad) == 0, f"seed.{f} differs at {bad[:8]}: got {got[f][bad[:8]]} want {want[f][bad[:8]]}"
        bad = np.nonzero(got["stable"] != want["stable"])[0]
        assert len(bad) == 0, f"seed.stable differs at {bad[:8]}"
    bad = np.nonzero(got["fused"] != want["fused"])[0]
    assert len(bad) == 0, f"seed.fused differs at {bad[:8]}"
    ng = np.stack([got["norm_x"], got["norm_y"], got["norm_z"]], -1).astype(np.float64)
    nw = np.stack([want["norm_x"], want["norm_y"], want["norm_z"]], -1).astype(np.float64)
    pg = np.stack([got["posi_x"], got["posi_y"], got["posi_z"]], -1).astype(np.float64)
    pw = np.stack([want["posi_x"], want["posi_y"], want["posi_z"]], -1).astype(np.float64)
    nanw = np.isnan(nw).any(1) | np.isnan(pw).any(1)
    nang = np.isnan(ng).any(1) | np.isnan(pg).any(1)
    assert (nanw == nang).all(), "seed NaN pattern differs"
    ok = ~nanw
    zero_w = (nw == 0).all(1)
    zero_g = (ng == 0).all(1)
    assert (zero_w[ok] == zero_g[ok]).all(), f"plane-fit accept/reject differs at {np.nonzero(ok & (zero_w != zero_g))[0][:8]}"
    # a seed the plane fit rejected keeps the mean_depth of the last Huber-Newton pass: clustering state, bit-exact
    if cluster_exact:
        rej = np.nonzero(ok & zero_w)[0]
        bad = rej[~bits_equal_nan(got["mean_depth"][rej], want["mean_depth"][rej])]
        assert len(bad) == 0, (f"seed.mean_depth of rejected seeds differs at {bad[:8]}: "
                               f"got {got['mean_depth'][bad[:8]]} want {want['mean_depth'][bad[:8]]}")
    assert np.linalg.norm(ng[ok] - nw[ok], axis=1).max() <= tol, "seed normal error"
    pe = np.linalg.norm(pg[ok] - pw[ok], axis=1) / np.maximum(np.linalg.norm(pw[ok], axis=1), 1e-12)
    assert pe.max() <= tol, f"seed position error {pe.max():.3e}"
    for f in ("view_cos", "mean_depth", "size"):
        g = got[f][ok].astype(np.float64)
        w = want[f][ok].astype(np.float64)
        err = np.abs(g - w) / np.maximum(np.abs(w), 1e-6)
        assert err.max() <= tol, f"seed.{f} error {err.max():.3e}"


def compact_like_caller(local, new):
    """What SurfelMap::fuse_map does after the call (surfel_map.cpp:1077-1109), as a set:
    drop dead surfels, add the new ones.  Same helper is applied to oracle and GPU results."""
    keep = local[local["update_times"] > 0] if len(local) else np.zeros(0, SURFEL_DTYPE)
    return np.concatenate([keep, new])


def canon(a):
    """field-by-field bytes (struct padding excluded) with every NaN canonicalised: NaN payload/sign
    and padding bytes are not part of the contract."""
    parts = []
    for f in a.dtype.names:
        v = np.ascontiguousarray(a[f]).copy()
        if v.dtype.kind == "f":
            v[np.isnan(v)] = np.float32(np.nan)
        parts.append(v.tobytes())
    return b"".join(parts)


def crc(x):
    return zlib.crc32(x if isinstance(x, (bytes, bytearray)) else np.ascontiguousarray(x).tobytes()) & 0xFFFFFFFF


def match_as_sets(got, want, tol=1e-4):
    """Pools are equal as sets: same size, and a one-to-one nearest-neighbour matching within tolerance."""
    assert len(got) == len(want), f"pool size {len(got)} != {len(want)}"
    if len(got) == 0:
        return
    key = lambda a: np.lexsort((a["pz"], a["py"], a["px"], a["last_update"], a["update_times"]))
    g, w = got[key(got)], want[key(want)]
    # lexsort on floats can differ in the last bits; repair by nearest neighbour inside equal-integer groups
    pg = np.stack([g["px"], g["py"], g["pz"]], -1).astype(np.float64)
    pw = np.stack([w["px"], w["py"], w["pz"]], -1).astype(np.float64)
    bad = np.nonzero(np.linalg.norm(pg - pw, axis=1) > tol * np.maximum(np.linalg.norm(pw, axis=1), 1.0))[0]
    if len(bad):
        used = set()
        for i in bad:
            dist = np.linalg.norm(pw[bad] - pg[i], axis=1)
            j = int(np.argmin(dist))
            assert dist[j] <= tol * max(np.linalg.norm(pg[i]), 1.0) and j not in used, f"surfel {i} has no partner"
            used.add(j)
            g[i], w_i = g[i], w[bad[j]]
            check_surfels(g[i:i + 1], np.array([w_i]), "set member")
        ok = np.setdiff1d(np.arange(len(g)), bad)
        check_surfels(g[ok], w[ok], "pool (sorted)")
    else:
        check_surfels(g, w, "pool (sorted)")


def random_surfels(n, seed=0):
    rng = np.random.RandomState(seed)
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz"):
        s[f] = rng.uniform(-40, 40, n)
    nr = rng.normal(size=(n, 3))
    nr /= np.linalg.norm(nr, axis=1, keepdims=True)
    s["nx"], s["ny"], s["nz"] = nr[:, 0], nr[:, 1], nr[:, 2]
    s["size"] = rng.uniform(0.01, 0.6, n)
    s["color"] = rng.randint(0, 256, n) + rng.choice([0.0, 0.25, 0.75], n)  # averaged intensities are not integers
    s["weight"] = rng.uniform(0.01, 30, n)
    s["update_times"] = rng.randint(0, 12, n)
    s["last_update"] = rng.randint(0, 9, n)
    if n >= 4:
        s["nx"][0], s["ny"][0], s["nz"][0] = 0, 0, 1    # x_dir = 0: normalize() must leave it alone, not make NaN
        s["nx"][1], s["ny"][1], s["nz"][1] = 1, 0, 0
        s["px"][2], s["py"][2], s["pz"][2] = 1e-7, -123456.78, 3.0e5  # exponent formats in %g
        s["size"][3] = 0
    return s


def canon_points(p):
    p = np.array(p, np.float32, copy=True)
    p[np.isnan(p)] = np.float32(np.nan)
    return p.tobytes()


# ---- the reference's SurfelMap ----
def poststep_frames():
    for t in range(4):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(CAM, 50 + t, pose)
        yield t + (7 if t == 3 else 0), gray, depth, pose  # the jump kills unstable surfels: slot recycling AND swap-with-back both run


def neighbor_replay(m, steps=8):
    """A controlled drive of the reference node with drift_free_poses=1: one keyframe per step, each referencing the
    previous one, a loop edge 4-0 at step 5 (pose 0 joins the neighbourhood of pose 4) and a return to pose 0 at step 7
    (pose 0 re-enters the drift-free window).  Yields, per step, after the pose feed: the pool before move_add_surfels,
    the window before and after it, the BFS list of publish_neighbor_pointcloud and what that publisher sent; then
    fuses the step's frame (fuse_map) for the next step."""
    path = []
    for t in range(steps):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(CAM, 1000 + t, pose)
        p7 = pyoracle.pose_to_ros7(pose)
        ref = 0 if t == steps - 1 else max(t - 1, 0)
        m.frame(100.0 + 0.1 * t, None, None, p7, True, ref, path7=np.array(path).reshape(-1, 7), loops=[4, 0] if t == 5 else ())
        path.append(p7)
        pool, window_before = m.local(), m.local_pose_indexs()
        m.move_add_surfels(ref)
        m.publish_clouds(ref)
        yield dict(t=t, ref=ref, pool=pool, window_before=window_before, window=m.local_pose_indexs(),
                   bfs=m.driftfree_poses(ref, 2), published=m.published("neighbor_pointcloud"))
        m.fuse_map(gray, depth, pose, ref)
