"""oracle/pyoracle_field_signed.py (the signed distance field of DESIGN.md §8.16) pinned against independent
restatements: a brute-force minimum over the complement on small plain and known grids, scipy's EDT of both sets, the
identities include/dsm.h states, axes of one voxel, all-site and no-site grids, the complement of every crafted pattern
of tests/edt_patterns.py, and the signed queries against scipy's linear map_coordinates in fp64."""
import numpy as np
import pytest
from scipy import ndimage

import edt_patterns as P
import pyoracle_field
import pyoracle_field_query as fq
import pyoracle_field_signed as fs

UNKNOWN, OCCUPIED, FREE = 0, 1, 2


def brute(sites, voxel):
    """sdist by brute force: per site the smallest squared distance to any voxel of F, per voxel of F to any site."""
    idx = np.argwhere(np.ones(sites.shape, bool))
    d2 = ((idx[:, None, :] - idx[None, :, :]) ** 2).sum(-1)
    s = sites.reshape(-1)
    out = np.empty(len(idx), np.float32)
    v = np.float32(voxel)
    for i in range(len(idx)):
        other = d2[i][~s] if s[i] else d2[i][s]
        if len(other) == 0:
            out[i] = -np.inf if s[i] else np.inf
        elif s[i]:
            out[i] = (np.float32(1) - np.sqrt(np.float32(other.min()))) * v
        else:
            out[i] = np.sqrt(np.float32(other.min())) * v
    return out.reshape(sites.shape)


def check_identities(sites, dist, sdist):
    e2 = pyoracle_field.squared_distances(~sites) if (~sites).any() else None
    assert (sdist <= dist).all()
    assert sdist[~sites].tobytes() == dist[~sites].tobytes()
    if e2 is not None:
        one = sites & (e2 == 1)
        assert sdist[one].tobytes() == dist[one].tobytes()
        assert ((sdist < 0) == (sites & (e2 >= 2))).all()


@pytest.mark.parametrize("seed", range(6))
def test_plain_grids_equal_the_brute_force_minimum(seed):
    rng = np.random.default_rng(seed)
    shape = tuple(int(n) for n in rng.integers(1, 8, 3))
    voxel = [0.1, 0.125, 0.3][seed % 3]
    o = np.array([-(n // 2) for n in shape])
    pts = (o + rng.random((int(rng.integers(1, 40)), 3)) * np.array(shape)) * np.float64(np.float32(voxel))
    dist, sdist, origin, n_occ = fs.field(pts.astype(np.float32), voxel, shape, (o + np.array(shape) // 2 + 0.5) * np.float64(np.float32(voxel)))
    occ = pyoracle_field.occupancy(pts.astype(np.float32), voxel, shape, origin.astype(np.int64))
    assert int(occ.sum()) == n_occ
    assert sdist.tobytes() == brute(occ, voxel).tobytes()
    check_identities(occ, dist, sdist)


@pytest.mark.parametrize("seed", range(6))
def test_known_grids_equal_the_brute_force_minimum(seed):
    rng = np.random.default_rng(100 + seed)
    shape = tuple(int(n) for n in rng.integers(1, 8, 3))
    state = rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1], p=[0.4, 0.1, 0.5]).astype(np.uint8)
    dist, sdist = fs.state_field(state, 0.2)
    sites = state != FREE
    assert sdist.tobytes() == brute(sites, 0.2).tobytes()
    check_identities(sites, dist, sdist)


@pytest.mark.parametrize("seed", range(4))
def test_against_scipy_edt_of_both_sets(seed):
    rng = np.random.default_rng(200 + seed)
    shape = (40, 31, 17)
    voxel = 0.2
    sites = rng.random(shape[::-1]) < [0.05, 0.3, 0.6, 0.95][seed]
    dist = (ndimage.distance_transform_edt(~sites) * voxel).astype(np.float32)
    sdist = fs.signed(sites, dist, voxel)
    want = np.where(sites, (1.0 - ndimage.distance_transform_edt(sites)) * voxel, ndimage.distance_transform_edt(~sites) * voxel)
    np.testing.assert_allclose(sdist, want, rtol=4e-7, atol=4e-7)
    check_identities(sites, dist, sdist)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 9, 1), (9, 1, 1), (1, 1, 9), (1, 6, 5), (6, 1, 5), (6, 5, 1)])
def test_axes_of_one_voxel(shape):
    rng = np.random.default_rng(sum(shape))
    for k in range(6):
        state = rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1]).astype(np.uint8)
        dist, sdist = fs.state_field(state, 0.125)
        assert sdist.tobytes() == brute(state != FREE, 0.125).tobytes()


@pytest.mark.parametrize("shape", [(1, 1, 1), (5, 4, 3)])
def test_all_sites_and_no_sites(shape):
    for s in (UNKNOWN, OCCUPIED):
        dist, sdist = fs.state_field(np.full(shape[::-1], s, np.uint8), 0.1)
        assert (dist == 0).all() and np.isneginf(sdist).all()
    dist, sdist = fs.state_field(np.full(shape[::-1], FREE, np.uint8), 0.1)
    assert np.isposinf(dist).all() and np.isposinf(sdist).all()


@pytest.mark.parametrize("name", list(P.PLANES))
def test_complement_of_every_crafted_pattern(name):
    """The pattern's sites become F: the signed pass along each plane sees the pattern's envelope, and every site's
    depth equals (1 - the pattern's own distance) * v."""
    n = 64
    shape = (n, n, 2)
    plane = P.PLANES[name](n) if name != "fan" else P.fan(n, 5)
    F = np.zeros((2, n, n), bool)
    F[...] = plane[:, :]          # [z][y][x]: b = y, a = x
    sites = ~F
    voxel = 0.1
    e2F = pyoracle_field.squared_distances(F)          # to F, which is the pattern
    dist = np.where(sites, np.float32(0), np.float32(np.inf)).astype(np.float32)   # sdist reads dist only on F
    sdist = fs.signed(sites, dist, voxel)
    want = np.where(sites, (np.float32(1) - np.sqrt(e2F.astype(np.float32))) * np.float32(voxel), np.float32(np.inf))
    assert sdist.tobytes() == want.astype(np.float32).tobytes()
    if name == "corner":   # one voxel of F per plane: the far corner is the deepest site
        assert sdist.min() == (np.float32(1) - np.sqrt(np.float32(2 * (n - 1) ** 2))) * np.float32(voxel)


# ---- signed queries ----
def gradient(s):
    return np.stack([s["gx"], s["gy"], s["gz"]], 1)


def test_signed_samples_are_linear_interpolation_within_fp32_rounding():
    rng = np.random.default_rng(7)
    shape, voxel = (23, 17, 9), 0.2
    state = rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1], p=[0.3, 0.1, 0.6]).astype(np.uint8)
    _, sdist = fs.state_field(state, voxel)
    origin = np.array([-5, 2, 7])
    u = rng.random((4000, 3)) * (np.array(shape) - 1)
    p = (u + origin + 0.5) * np.float64(np.float32(voxel))
    got = fs.sample(sdist, origin, voxel, p)
    want = ndimage.map_coordinates(sdist.astype(np.float64), [u[:, 2], u[:, 1], u[:, 0]], order=1, mode="nearest")
    assert np.isfinite(got["dist"]).all() and (got["dist"] < 0).any()
    np.testing.assert_allclose(got["dist"], want, rtol=0, atol=8 * np.finfo(np.float32).eps * np.abs(sdist).max())


def test_gradient_deep_in_unknown_space_points_to_the_free_side():
    """Free for x < 8, unknown beyond: the unsigned field is 0 with a zero gradient deep inside, the signed one falls by
    one voxel edge per voxel and its gradient is (-1, 0, 0)."""
    shape, voxel = (24, 6, 5), 0.1
    state = np.full(shape[::-1], UNKNOWN, np.uint8)
    state[:, :, :8] = FREE
    dist, sdist = fs.state_field(state, voxel)
    origin = np.zeros(3, np.int64)
    p = (np.array([[15.3, 2.5, 2.2]]) + 0.5) * np.float64(np.float32(voxel))
    pos = fq.sample(dist, origin, voxel, p)[0]
    neg = fs.sample(sdist, origin, voxel, p)[0]
    assert pos["dist"] == 0 and (pos["gx"], pos["gy"], pos["gz"]) == (0, 0, 0)
    assert neg["dist"] < -0.6 and neg["gx"] < 0 and neg["gy"] == 0 and neg["gz"] == 0
    np.testing.assert_allclose(neg["gx"], -1.0, rtol=1e-5)


def test_clearance_with_negative_minima_and_the_infinity_rules():
    shape, voxel = (24, 6, 5), 0.1
    v = np.float64(np.float32(voxel))
    state = np.full(shape[::-1], UNKNOWN, np.uint8)
    state[:, :, :8] = FREE
    _, sdist = fs.state_field(state, voxel)
    o = np.zeros(3, np.int64)
    wp = np.array([[1.5, 2.5, 2.5], [20.5, 2.5, 2.5], [3.5, 1.5, 1.5], [6.5, 4.5, 3.5]]) * v
    ofs = np.array([0, 2, 4], np.int32)
    c = fs.clearance(sdist, o, voxel, wp, ofs, 0.05, 0.0)
    # the first path enters the unknown side: its deepest sample is its last waypoint, 20 - 7 voxels from F
    assert c["min_dist"][0] == (np.float32(1) - np.sqrt(np.float32(13 ** 2))) * np.float32(voxel)
    assert c["first_hit"][0] >= 0 and c["argmin"][0] > c["first_hit"][0]
    assert c["min_dist"][1] > 0 and c["first_hit"][1] == -1
    # every voxel a site: -inf at every inside sample, the first one is both the minimum and the first hit
    full = np.full(shape[::-1], -np.inf, np.float32)
    c = fs.clearance(full, o, voxel, wp, ofs, 0.05, 0.0)
    assert np.isneginf(c["min_dist"]).all() and (c["argmin"] == 0).all() and (c["first_hit"] == 0).all()
    s = fs.sample(full, o, voxel, np.vstack([wp, [[1e9, 0, 0]]]))
    assert np.isneginf(s["dist"][:-1]).all() and np.isnan(s["dist"][-1]) and (gradient(s) == 0).all()
    # no site: +inf
    free = np.full(shape[::-1], np.inf, np.float32)
    s = fs.sample(free, o, voxel, wp)
    assert np.isposinf(s["dist"]).all() and (gradient(s) == 0).all()
