"""oracle/pyoracle_trajectory.py (the trajectory job of DESIGN.md §8.17) pinned against independent restatements: each
cost term's gradient against central differences on an analytic field and on trilinear grids, the B-spline basis at the
knots, the warp reduction against a plain loop, scipy's L-BFGS-B on the smoothness term alone, hand cases on crafted
state grids (a pillar, a wall with a gap, an over-fast path, a path through deep unknown space), every status,
max_iter = 0 and every refusal."""
import numpy as np
import pytest
from scipy import optimize

import pyoracle_field_signed as fs
import pyoracle_trajectory as tj

UNKNOWN, OCCUPIED, FREE = 0, 1, 2


def sphere_sampler(c, R):
    """An analytic smooth field: the signed distance to a sphere of radius R at c, and its gradient."""
    c = np.asarray(c, np.float64)

    def sampler(p):
        d = p - c
        r = np.sqrt((d * d).sum(1))
        return np.ones(len(p), bool), r - R, d / r[:, None]
    return sampler


def cost(Q, dt, p, sampler):
    return tj.evaluate(Q, dt, p, sampler)[0]


def fd_gradient(Q, dt, p, sampler, h):
    g = np.zeros((len(Q) - 6, 3))
    for i in range(3, len(Q) - 3):
        for k in range(3):
            a, b = Q.copy(), Q.copy()
            a[i, k] += h
            b[i, k] -= h
            g[i - 3, k] = (cost(a, dt, p, sampler) - cost(b, dt, p, sampler)) / (2 * h)
    return g


def line(n, a=(0.0, 0.0, 0.0), b=(4.0, 0.0, 0.0)):
    t = np.linspace(0, 1, n)[:, None]
    return np.asarray(a, np.float64) + t * (np.asarray(b, np.float64) - np.asarray(a, np.float64))


def padded(path):
    """A path's points with the start and end repeated three times, as INTEGRATION.md §4 builds initial points."""
    path = np.asarray(path, np.float64)
    return np.concatenate([path[:1], path[:1], path, path[-1:], path[-1:]])


# ---- the building blocks ----
def test_reduce_is_lane_sums_and_a_butterfly():
    rng = np.random.default_rng(0)
    for n in (1, 5, 31, 32, 33, 64, 250):
        v = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
        lanes = [0.0] * 32
        for k in range(n):
            lanes[k % 32] = lanes[k % 32] + v[k]
        for m in (16, 8, 4, 2, 1):
            lanes = [lanes[l] + lanes[l ^ m] for l in range(32)]
        assert len({x.hex() for x in lanes}) == 1
        assert tj.reduce(v) == lanes[0]


def test_basis_at_the_knots():
    rng = np.random.default_rng(1)
    Q = rng.standard_normal((12, 3)) * 5
    K = 4
    pts = tj.curve_samples(Q, K)
    assert len(pts) == (12 - 3) * K + 1
    for m in range(12 - 3):
        want = (Q[m] + 4 * Q[m + 1] + Q[m + 2]) / 6
        np.testing.assert_allclose(pts[m * K], want, rtol=0, atol=1e-13)
    np.testing.assert_allclose(pts[-1], (Q[-3] + 4 * Q[-2] + Q[-1]) / 6, rtol=0, atol=1e-13)
    assert sum(tj.basis(0.37)) == pytest.approx(1.0, abs=1e-15)


@pytest.mark.parametrize("term", ["smooth", "clear", "feas", "all"])
def test_gradient_against_central_differences_on_an_analytic_field(term):
    rng = np.random.default_rng(2)
    Q = line(14, (-2, 0.3, 0.1), (2, -0.2, 0.4)) + rng.standard_normal((14, 3)) * 0.2
    w = dict(smooth=(1, 0, 0), clear=(0, 1, 0), feas=(0, 0, 1), all=(1, 3, 0.5))[term]
    p = tj.params(*w, margin=1.5, v_max=0.5, a_max=0.5)
    s = sphere_sampler((0.1, 0.2, -0.3), 0.6)
    J, _, g, _ = tj.evaluate(Q, 0.4, p, s)
    assert J > 0
    np.testing.assert_allclose(g, fd_gradient(Q, 0.4, p, s, 1e-6), rtol=1e-6, atol=1e-6 * max(1.0, np.abs(g).max()))


def test_clearance_gradient_against_central_differences_on_a_trilinear_grid():
    rng = np.random.default_rng(3)
    shape, voxel, origin = (24, 20, 12), 0.2, np.array([-12, -10, -6])
    st = np.full(shape[::-1], FREE, np.uint8)
    st[4:8, 8:12, 10:14] = OCCUPIED
    st[:, :3, :] = UNKNOWN
    _, sdist = fs.state_field(st, voxel)
    s = tj.grid_sampler(sdist, origin, voxel)
    v = np.float64(np.float32(voxel))
    # free points at fractions 0.3 .. 0.7 within their cells: away from the faces, where the interpolant is smooth
    cells = rng.integers(2, np.array(shape) - 3, (10, 3))
    Q = (cells + origin + 0.5 + rng.uniform(0.3, 0.7, (10, 3))) * v
    p = tj.params(0, 1, 0, margin=1.0)
    _, (_, Jc, _), g, _ = tj.evaluate(Q, 0.5, p, s)
    assert Jc > 0
    np.testing.assert_allclose(g, fd_gradient(Q, 0.5, p, s, 1e-4 * v), rtol=0, atol=2e-3 * max(1.0, np.abs(g).max()))


# ---- hand cases ----
def free_grid(shape=(64, 32, 32), voxel=0.1):
    return np.full(shape[::-1], FREE, np.uint8), voxel


def run(Q, dt, p, state, voxel, origin):
    _, sdist = fs.state_field(state, voxel)
    Q = np.asarray(Q, np.float64)
    out, rec, info = tj.job(Q, [0, len(Q)], [dt], p, sdist, origin, voxel)
    return out, rec[0], info, sdist


def test_evenly_spaced_collinear_points_return_at_iteration_zero():
    st, voxel = free_grid()
    st[0, 0, 0] = OCCUPIED   # one far site: the path is clear by more than the margin
    origin = np.array([-32, -16, -16])
    Q = np.zeros((20, 3))
    Q[:, 0], Q[:, 1] = np.arange(20) * 0.25 - 2.0, 0.0625   # exact steps: every jerk term is 0
    out, r, info, _ = run(Q, 1.0, tj.params(margin=0.3, v_max=5, a_max=5), st, voxel, origin)
    assert r["status"] == 0 and r["iterations"] == 0 and r["evaluations"] == 1
    assert out.tobytes() == Q.tobytes() and r["cost"] == r["cost_start"] == 0.0
    assert info["n_status"].tolist() == [1, 0, 0, 0]


def test_smoothness_alone_reaches_scipys_optimum():
    rng = np.random.default_rng(4)
    Q = line(16, (0, 0, 0), (3, 1, -1)) + rng.standard_normal((16, 3)) * 0.3
    p = tj.params(1, 0, 0, g_tol=1e-9, max_iter=1000, memory=16)
    st, voxel = free_grid()
    out, r, _, _ = run(Q, 1.0, p, st, voxel, np.array([-32, -16, -16]))
    assert r["status"] in (0, 2)   # 2: the Armijo test can no longer tell J apart in fp64

    def f(z):
        X = Q.copy()
        X[3:-3] = z.reshape(-1, 3)
        j = tj.jerk(X)
        return (j * j).sum()
    ref = optimize.minimize(f, Q[3:-3].reshape(-1), method="L-BFGS-B", options=dict(ftol=1e-15, gtol=1e-12, maxiter=10000))
    assert r["cost"] == pytest.approx(ref.fun, rel=1e-9)
    np.testing.assert_allclose(out[3:-3].reshape(-1), ref.x, atol=1e-4)


def pillar_grid():
    st = np.full((16, 40, 80), FREE, np.uint8)       # z, y, x
    st[:, 18:22, 38:42] = OCCUPIED                    # a 4 x 4 voxel pillar through the whole height
    return st, 0.1, np.array([-40, -20, -8])


def test_a_path_through_a_pillar_clears_it():
    st, voxel, origin = pillar_grid()
    Q = padded(line(24, (-3.0, 0.15, 0.0), (3.0, 0.15, 0.0)))   # grazing the pillar's +y half
    p = tj.params(1, 50, 1, margin=0.4, v_max=10, a_max=10, max_iter=300, memory=8, radius=0.2)
    out, r, _, sdist = run(Q, 0.5, p, st, voxel, origin)
    assert tj.final_check(Q, 0.5, p["samples"], p["radius"], sdist, origin, voxel)[2] >= 0   # it hit before
    assert r["min_dist"] >= 0.4 - 0.05 and r["first_hit"] == -1
    assert r["cost"] < r["cost_start"]


def test_a_path_through_a_wall_with_a_gap_centres_in_the_gap():
    st = np.full((24, 40, 80), FREE, np.uint8)
    st[:, :, 39:41] = OCCUPIED                         # a wall across x
    st[8:16, 16:24, 39:41] = FREE                      # an 8 x 8 voxel gap
    voxel, origin = 0.1, np.array([-40, -20, -12])
    Q = padded(line(18, (-3.0, -0.32, 0.1), (3.0, -0.32, 0.1)))   # through the gap, clipping its edge
    p = tj.params(1, 50, 1, margin=0.3, v_max=10, a_max=10, max_iter=300, radius=0.15)
    out, r, _, sdist = run(Q, 0.5, p, st, voxel, origin)
    assert tj.final_check(Q, 0.5, p["samples"], p["radius"], sdist, origin, voxel)[2] >= 0   # it hit before
    assert r["first_hit"] == -1 and r["min_dist"] >= 0.15


def test_an_over_fast_trajectory_comes_within_the_limits():
    st, voxel = free_grid()
    rng = np.random.default_rng(5)
    Q = padded(line(16, (-1.0, 0, 0), (1.0, 0, 0)))
    Q[4:-4] += rng.standard_normal((len(Q) - 8, 3)) * 0.4   # zig-zags far faster than the straight line needs
    p = tj.params(0.01, 0, 10, v_max=1.0, a_max=4.0, max_iter=500, memory=16, g_tol=1e-9)
    out, r, _, _ = run(Q, 0.3, p, st, voxel, np.array([-32, -16, -16]))
    _, _, _, _, v0, _ = tj.final_check(Q, 0.3, 4, 0.1, *fs.state_field(st, voxel)[1:], np.array([-32, -16, -16]), voxel)
    assert v0 > 2.0
    assert r["max_v"] <= 1.0 * 1.1 and r["max_a"] <= 4.0 * 1.1


def test_a_path_through_deep_unknown_space_moves_out_of_it():
    """A block of unknown space beside a free corridor: the signed grid pushes the path out; on the unsigned grid the
    points deep inside the block have no clearance gradient at all."""
    st = np.full((24, 40, 80), FREE, np.uint8)
    st[:, 14:40, 30:50] = UNKNOWN
    voxel, origin = 0.1, np.array([-40, -20, -12])
    Q = padded(line(18, (-3.0, 0.2, 0.0), (3.0, 0.2, 0.0)))   # 0.6 m deep inside the unknown block at its middle
    p = tj.params(1, 50, 1, margin=0.2, v_max=10, a_max=10, max_iter=300)
    dist, sdist = fs.state_field(st, voxel)
    out, rec, _ = tj.job(Q, [0, len(Q)], [0.5], p, sdist, origin, voxel)
    before = tj.final_check(Q, 0.5, p["samples"], p["radius"], sdist, origin, voxel)[0]
    assert before < -0.4 and rec[0]["min_dist"] > before + 0.4
    deep = np.abs(Q[3:-3, 0]) < 0.5
    c = tj.params(0, 1, 0, margin=0.2)
    assert (tj.evaluate(Q, 0.5, c, tj.grid_sampler(dist, origin, voxel))[2][deep] == 0).all()
    assert (tj.evaluate(Q, 0.5, c, tj.grid_sampler(sdist, origin, voxel))[2][deep][:, 1] > 0).all()


# ---- statuses and parameters ----
def test_statuses():
    st, voxel = free_grid()
    st[:, :, :20] = OCCUPIED
    origin = np.array([-32, -16, -16])
    rng = np.random.default_rng(6)
    Q = padded(line(10, (-1.0, 0, 0), (1.0, 0, 0))) + 0
    Q[4:-4] += rng.standard_normal((len(Q) - 8, 3)) * 0.2
    # 1: out of iterations
    _, r, _, _ = run(Q, 1.0, tj.params(max_iter=2), st, voxel, origin)
    assert r["status"] == 1 and r["iterations"] == 2
    # max_iter = 0 only evaluates
    out, r, _, _ = run(Q, 1.0, tj.params(max_iter=0), st, voxel, origin)
    assert r["status"] == 1 and r["iterations"] == 0 and r["evaluations"] == 1 and r["cost"] == r["cost_start"]
    assert out.tobytes() == Q.tobytes()
    # 2: a stiff problem whose one-voxel first step overshoots, with one trial
    big = np.full((8, 8, 8), FREE, np.uint8)
    Qs = line(12, (0, 0, 0), (1, 1, 1)) + rng.standard_normal((12, 3)) * 1e-4
    out, rec, _ = tj.job(Qs, [0, 12], [1.0], tj.params(1e6, 0, 0, max_ls=1), fs.state_field(big, 1.0)[1], (-4, -4, -4), 1.0)
    assert rec[0]["status"] == 2 and rec[0]["iterations"] == 0 and out.tobytes() == Qs.tobytes()
    # 3: no voxel of F
    unk = np.full((8, 8, 8), UNKNOWN, np.uint8)
    out, rec, info = tj.job(Qs, [0, 12], [1.0], tj.params(), fs.state_field(unk, 1.0)[1], (-4, -4, -4), 1.0)
    assert rec[0]["status"] == 3 and rec[0]["evaluations"] == 0 and rec[0]["cost_start"] == 0 and out.tobytes() == Qs.tobytes()
    assert rec[0]["min_dist"] == -np.inf and info["n_status"].tolist() == [0, 0, 0, 1]


def test_points_outside_the_grid_are_counted_and_contribute_nothing():
    st, voxel = free_grid((16, 16, 16), 0.1)
    st[:, :, :4] = OCCUPIED
    Q = line(12, (-0.5, 0, 0), (3.0, 0, 0))   # the grid spans [-0.8, 0.8): the last free points lie outside
    _, sdist = fs.state_field(st, voxel)
    J, _, g, nout = tj.evaluate(Q, 1.0, tj.params(0, 1, 0, margin=5.0), tj.grid_sampler(sdist, (-8, -8, -8), voxel))
    assert nout > 0 and (g[-nout:] == 0).all() and (g[:-nout] != 0).any()


def test_refusals():
    Q = line(8)
    p = tj.params()
    tj.check_request(Q, [0, 8], [1.0], p)
    bad = [
        (Q, [0, 6], [1.0], p),                                   # N < 7
        (line(257), [0, 257], [1.0], p),                         # N > 256
        (Q, [1, 8], [1.0], p),                                   # offsets[0] != 0
        (np.concatenate([Q, Q]), [0, 8, 7], [1.0, 1.0], p),      # offsets that do not rise
        (np.where(np.arange(24).reshape(8, 3) == 5, np.nan, Q), [0, 8], [1.0], p),
        (Q, [0, 8], [0.0], p), (Q, [0, 8], [np.inf], p),
        (Q, [0, 8], [1.0], tj.params(w_clear=-1)), (Q, [0, 8], [1.0], tj.params(margin=np.nan)),
        (Q, [0, 8], [1.0], tj.params(max_iter=1025)), (Q, [0, 8], [1.0], tj.params(max_iter=-1)),
        (Q, [0, 8], [1.0], tj.params(memory=0)), (Q, [0, 8], [1.0], tj.params(memory=17)),
        (Q, [0, 8], [1.0], tj.params(max_ls=0)), (Q, [0, 8], [1.0], tj.params(max_ls=33)),
        (Q, [0, 8], [1.0], tj.params(samples=0)), (Q, [0, 8], [1.0], tj.params(samples=65)),
        (Q, [0, 8], [1.0], tj.params(radius=-1)),
    ]
    for args in bad:
        with pytest.raises(ValueError):
            tj.check_request(*args)
    # the work bounds: 2^32 field samples of optimisation, 2^26 final samples
    n = 1 << 12
    big = np.zeros((256 * n, 3))
    ofs = np.arange(n + 1) * 256
    tj.check_request(big, ofs, np.ones(n), tj.params(max_iter=1024, max_ls=3, samples=64))
    with pytest.raises(ValueError):
        tj.check_request(big, ofs, np.ones(n), tj.params(max_iter=1024, max_ls=4))
    n2 = (1 << 26) // (253 * 64) + 1
    with pytest.raises(ValueError):
        tj.check_request(np.zeros((256 * n2, 3)), np.arange(n2 + 1) * 256, np.ones(n2), tj.params(max_iter=0, samples=64))
