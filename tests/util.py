"""Shared comparison helpers for the parity tests (tolerances from BASELINE.json north_star /
SURVEY.md §7 H5: labels and the clustering state bit-exact, surfel geometry within 1e-4 using
norm-based metrics, integer fields exact, NaN == NaN)."""
import numpy as np

from densesurfelmapping_b200.elements import SURFEL_DTYPE

TOL = 1e-4


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
