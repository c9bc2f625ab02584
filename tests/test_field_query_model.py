"""oracle/pyoracle_field_query.py (the planner queries of DESIGN.md §8.8) pinned against independent restatements: scipy's
linear map_coordinates in fp64, finite differences of the interpolant, exact values at voxel centres, the inside rule at
the grid's last centre, axes of one voxel, the empty field, non-finite points, a plain Python loop for the trajectory
clearance and every request the library refuses."""
import math

import numpy as np
import pytest
from scipy import ndimage

import pyoracle_field
import pyoracle_field_query as fq


def random_field(rng, shape, voxel):
    """A real field of random obstacles: dist float32 [nz][ny][nx] and an origin."""
    nx, ny, nz = shape
    o = np.array([-(nx // 2), 3 - ny // 2, -1], np.int64)
    pts = (o + rng.random((max(nx * ny * nz // 40, 1), 3)) * np.array(shape)) * np.float32(voxel)
    dist, origin, n_occ = pyoracle_field.field(pts.astype(np.float32), voxel, shape, (o + np.array(shape) // 2) * float(np.float32(voxel)))
    assert n_occ > 0 and origin.tolist() == o.tolist()
    return dist, origin


def grad(s):
    return np.stack([s["gx"], s["gy"], s["gz"]], 1)


def u_of(points, origin, voxel):
    return np.asarray(points, np.float64) / np.float64(np.float32(voxel)) - origin.astype(np.float64) - 0.5


def points_inside(rng, n, origin, voxel, shape):
    u = rng.random((n, 3)) * (np.array(shape) - 1)
    return (u + origin + 0.5) * np.float64(np.float32(voxel))


@pytest.mark.parametrize("voxel", [0.1, 0.125, 0.3])
def test_distance_is_linear_interpolation_within_fp32_rounding(voxel):
    rng = np.random.default_rng(1)
    shape = (23, 17, 9)
    dist, origin = random_field(rng, shape, voxel)
    p = points_inside(rng, 4000, origin, voxel, shape)
    got = fq.sample(dist, origin, voxel, p)
    u = u_of(p, origin, voxel)
    want = ndimage.map_coordinates(dist.astype(np.float64), [u[:, 2], u[:, 1], u[:, 0]], order=1, mode="nearest")
    assert np.isfinite(got["dist"]).all()
    np.testing.assert_allclose(got["dist"], want, rtol=0, atol=8 * np.finfo(np.float32).eps * dist.max())


def test_gradient_is_the_derivative_of_the_interpolant_inside_cells():
    rng = np.random.default_rng(2)
    shape, voxel = (15, 12, 10), 0.2
    dist, origin = random_field(rng, shape, voxel)
    d64 = dist.astype(np.float64)
    cell = rng.integers(0, np.array(shape) - 1, (500, 3))
    u = cell + 0.1 + 0.8 * rng.random((500, 3))           # away from the cell faces, where the interpolant is smooth
    p = (u + origin + 0.5) * np.float64(np.float32(voxel))
    got = fq.sample(dist, origin, voxel, p)
    h = 1e-4
    for k, name in enumerate(("gx", "gy", "gz")):
        e = np.zeros(3)
        e[k] = h
        up, dn = u + e, u - e
        f = [ndimage.map_coordinates(d64, [q[:, 2], q[:, 1], q[:, 0]], order=1) for q in (up, dn)]
        fd = (f[0] - f[1]) / (2 * h) / np.float64(np.float32(voxel))
        np.testing.assert_allclose(got[name], fd, rtol=1e-4, atol=1e-3 * dist.max() / voxel)


@pytest.mark.parametrize("voxel", [0.125, 0.25, 1.0])
def test_exact_values_at_voxel_centres(voxel):
    rng = np.random.default_rng(3)
    shape = (9, 8, 7)
    dist, origin = random_field(rng, shape, voxel)
    idx = np.indices(shape).reshape(3, -1).T                    # (x, y, z)
    p = (idx + origin + 0.5) * voxel                             # exact: the voxel edge is a power of two
    got = fq.sample(dist, origin, voxel, p)
    want = dist[idx[:, 2], idx[:, 1], idx[:, 0]]
    assert got["dist"].tobytes() == want.tobytes()


def test_the_last_centre_is_inside_and_the_next_double_is_not():
    voxel, shape = 0.125, (6, 5, 4)
    dist, origin = random_field(np.random.default_rng(4), shape, voxel)
    origin = np.zeros(3, np.int64)   # u = 8p - 0.5 is exact, so the next double above p gives the next u above n - 1
    for k in range(3):
        p = np.full((1, 3), 0.5 * voxel)
        p[0, k] = (shape[k] - 1 + 0.5) * voxel
        assert u_of(p, origin, voxel)[0, k] == shape[k] - 1
        inside = fq.sample(dist, origin, voxel, p)[0]
        corner = [0, 0, 0]
        corner[k] = shape[k] - 1
        assert inside["dist"] == dist[corner[2], corner[1], corner[0]]
        q = p.copy()
        q[0, k] = np.nextafter(p[0, k], np.inf)
        assert u_of(q, origin, voxel)[0, k] == np.nextafter(float(shape[k] - 1), np.inf)
        out = fq.sample(dist, origin, voxel, q)[0]
        assert out["dist"].view(np.uint32) == 0x7FC00000 and out["gx"] == out["gy"] == out["gz"] == 0
        r = np.full((1, 3), 0.5 * voxel)
        r[0, k] = np.nextafter(0.5 * voxel, -np.inf)             # just below u = 0
        assert np.isnan(fq.sample(dist, origin, voxel, r)[0]["dist"])


@pytest.mark.parametrize("shape", [(1, 1, 1), (4, 1, 3), (1, 6, 1)])
def test_axes_of_one_voxel(shape):
    voxel = 0.125
    rng = np.random.default_rng(5)
    dist = (rng.random(shape[::-1]) * 3).astype(np.float32)
    origin = np.array([2, -3, 0], np.int64)
    u = rng.random((300, 3)) * np.maximum(np.array(shape) - 1, 0)
    p = (u + origin + 0.5) * voxel
    got = fq.sample(dist, origin, voxel, p)
    assert not np.isnan(got["dist"]).any()
    want = ndimage.map_coordinates(dist.astype(np.float64), [u[:, 2], u[:, 1], u[:, 0]], order=1, mode="nearest")
    np.testing.assert_allclose(got["dist"], want, atol=1e-5)
    for k, name in enumerate(("gx", "gy", "gz")):
        if shape[k] == 1:
            assert (got[name] == 0).all()
            q = p.copy()
            q[:, k] += voxel * 1e-6                               # off the only centre of that axis: outside
            assert np.isnan(fq.sample(dist, origin, voxel, q)["dist"]).all()


def test_empty_field_and_non_finite_points():
    shape, voxel = (8, 7, 6), 0.2
    dist = np.full(shape[::-1], np.inf, np.float32)
    origin = np.array([-4, -3, -3], np.int64)
    rng = np.random.default_rng(6)
    p = points_inside(rng, 50, origin, voxel, shape)
    got = fq.sample(dist, origin, voxel, p)
    assert np.isposinf(got["dist"]).all() and (grad(got) == 0).all()
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e308, 0, 0], [-1e308, 0, 0], [0, 0, 5e300]])
    for d in (dist, random_field(rng, shape, voxel)[0]):
        out = fq.sample(d, origin, voxel, bad)
        assert (out["dist"].view(np.uint32) == 0x7FC00000).all()
        assert (grad(out) == 0).all()


# ---- trajectory clearance ----
def loop_clearance(dist, origin, voxel, waypoints, offsets, step, radius):
    """The definition sample by sample in plain Python floats."""
    out = []
    st = float(np.float32(step))
    for j in range(len(offsets) - 1):
        w = [tuple(float(c) for c in waypoints[i]) for i in range(offsets[j], offsets[j + 1])]
        pts = []
        for a, b in zip(w[:-1], w[1:]):
            dx, dy, dz = b[0] - a[0], b[1] - a[1], b[2] - a[2]
            m = max(1, math.ceil(math.sqrt((dx * dx + dy * dy) + dz * dz) / st))
            for s in range(m):
                f = s / m
                pts.append((a[0] + f * (b[0] - a[0]), a[1] + f * (b[1] - a[1]), a[2] + f * (b[2] - a[2])))
        pts.append(w[-1])
        best, arg, hit, outside = math.inf, -1, -1, 0
        for i, p in enumerate(pts):
            d = float(fq.sample(dist, origin, voxel, np.array([p]))["dist"][0])
            if math.isnan(d):
                outside += 1
                continue
            if arg < 0 or d < best:
                best, arg = d, i
            if hit < 0 and d < float(np.float32(radius)):
                hit = i
        out.append((np.float32(best), arg, hit, outside))
    return out


def as_tuples(c):
    return [(np.float32(r["min_dist"]), int(r["argmin"]), int(r["first_hit"]), int(r["n_outside"])) for r in c]


def trajectories(rng, origin, voxel, shape, n):
    """n trajectories of 1-7 waypoints in and around the box, with zero-length segments and one-waypoint trajectories."""
    lo = (origin - 2) * voxel
    hi = (origin + np.array(shape) + 2) * voxel
    wps, offsets = [], [0]
    for j in range(n):
        k = 1 if j % 5 == 0 else int(rng.integers(2, 8))
        w = lo + rng.random((k, 3)) * (hi - lo)
        if k > 2 and j % 3 == 0:
            w[1] = w[0]                                           # a zero-length segment
        wps.append(w)
        offsets.append(offsets[-1] + k)
    return np.concatenate(wps), np.array(offsets, np.int32)


@pytest.mark.parametrize("voxel", [0.1, 0.125])
def test_clearance_equals_a_plain_loop(voxel):
    rng = np.random.default_rng(7)
    shape = (20, 16, 10)
    dist, origin = random_field(rng, shape, voxel)
    wp, ofs = trajectories(rng, origin, voxel, shape, 40)
    for step, radius in ((voxel / 2, 2 * voxel), (0.37, 0.0), (3 * voxel, 100.0)):
        got = fq.clearance(dist, origin, voxel, wp, ofs, step, radius)
        assert as_tuples(got) == loop_clearance(dist, origin, voxel, wp, ofs, step, radius)
    assert (got["first_hit"] >= 0).any() and (got["n_outside"] > 0).any()


def test_clearance_ties_hits_and_edge_cases():
    voxel, shape = 0.25, (8, 8, 8)
    origin = np.zeros(3, np.int64)
    flat = np.full(shape[::-1], 0.5, np.float32)                 # every inside sample ties
    wp = np.array([[-1.0, 1, 1], [3.0, 1, 1],                     # starts outside, then inside
                   [1.0, 1, 1],                                   # one waypoint
                   [0.5, 0.5, 0.5], [0.5, 0.5, 0.5], [1.5, 0.5, 0.5],   # a zero-length segment first
                   [50.0, 50, 50], [60.0, 50, 50]])                # all outside
    ofs = np.array([0, 2, 3, 6, 8], np.int32)
    c = fq.clearance(flat, origin, voxel, wp, ofs, 0.25, 0.6)
    assert as_tuples(c) == loop_clearance(flat, origin, voxel, wp, ofs, 0.25, 0.6)
    outside = np.isnan(fq.sample(flat, origin, voxel, fq.trajectory_samples(wp[:2], [0, 2], 0.25)[0])["dist"])
    first_inside = int(np.argmax(~outside))
    assert first_inside > 0 and c[0]["argmin"] == first_inside and c[0]["first_hit"] == first_inside
    assert c[0]["n_outside"] == outside.sum() > first_inside                  # it leaves the box again
    assert tuple(c[1].tolist()) == (np.float32(0.5), 0, 0, 0)
    assert c[2]["argmin"] == 0 and c[2]["n_outside"] == 0
    assert np.isposinf(c[3]["min_dist"]) and c[3]["argmin"] == -1 and c[3]["first_hit"] == -1 and c[3]["n_outside"] == 41   # 10 m at 0.25 m, and the end
    assert (fq.clearance(flat, origin, voxel, wp, ofs, 0.25, 0.5)["first_hit"] == -1).all()   # dist < radius, strictly
    empty = np.full(shape[::-1], np.inf, np.float32)
    e = fq.clearance(empty, origin, voxel, wp, ofs, 0.25, 1e30)
    assert as_tuples(e) == loop_clearance(empty, origin, voxel, wp, ofs, 0.25, 1e30)
    assert np.isposinf(e["min_dist"]).all() and e[1]["argmin"] == 0 and (e["first_hit"] == -1).all()
    pts, traj, idx = fq.trajectory_samples(wp, ofs, 0.25)
    assert traj.tolist() == sorted(traj.tolist()) and (idx[traj == 1] == [0]).all()
    assert (pts[traj == 2][:2] == wp[3]).all()                    # the zero-length segment gives its start once


@pytest.mark.parametrize("bad", ["offsets_start", "offsets_flat", "offsets_beyond", "nan_waypoint", "inf_waypoint", "step_zero",
                                 "step_negative", "step_nan", "step_inf", "radius_negative", "radius_nan", "radius_inf",
                                 "too_many_samples", "overflowing_length"])
def test_every_refused_request(bad):
    wp = np.array([[0.0, 0, 0], [1, 0, 0], [1, 1, 0], [2, 2, 2]])
    ofs, step, radius = [0, 2, 4], 0.1, 0.2
    fq.check_request(wp, ofs, step, radius)
    fq.trajectory_samples(wp, ofs, step)
    if bad == "offsets_start":
        ofs = [1, 2, 4]
    elif bad == "offsets_flat":
        ofs = [0, 2, 2, 4]
    elif bad == "offsets_beyond":
        ofs = [0, 2, 5]
    elif bad == "nan_waypoint":
        wp[3, 1] = np.nan
    elif bad == "inf_waypoint":
        wp[0, 2] = -np.inf
    elif bad.startswith("step"):
        step = {"step_zero": 0.0, "step_negative": -0.1, "step_nan": np.nan, "step_inf": np.inf}[bad]
    elif bad.startswith("radius"):
        radius = {"radius_negative": -1e-30, "radius_nan": np.nan, "radius_inf": np.inf}[bad]
    elif bad == "too_many_samples":
        wp[1, 0] = fq.MAX_SAMPLES * step          # one segment of 2^26 samples, plus the end samples
    elif bad == "overflowing_length":
        wp[0, 0], wp[1, 0] = -1e200, 1e200         # finite waypoints, infinite length
    with pytest.raises(ValueError):
        fq.check_request(wp, ofs, step, radius)
        fq.segment_counts(*fq.check_request(wp, ofs, step, radius), step)


def test_sample_count_bound_is_inclusive():
    step = 0.5
    m = fq.MAX_SAMPLES - 1
    wp = np.array([[0.0, 0, 0], [m * step, 0, 0]])
    counts, _, _ = fq.segment_counts(*fq.check_request(wp, [0, 2], step, 0.0), step)
    assert counts.sum() == fq.MAX_SAMPLES
    wp[1, 0] = np.nextafter(m * step, np.inf)
    with pytest.raises(ValueError):
        fq.segment_counts(*fq.check_request(wp, [0, 2], step, 0.0), step)
