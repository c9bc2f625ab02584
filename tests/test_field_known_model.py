"""oracle/pyoracle_field_known, the definition of dsm_field_enqueue_known's known-space field: the ray walk against exact
geometry (fractions.Fraction of the fp64 inputs), hand-made rays at the edges of the definition (axis-aligned rays,
edges and corners, a ray inside one voxel, truncation, cameras and rays outside the grid, negative coordinates), the
state grid and the distance, the capture predicate, and every refused request.  tests/test_gpu_field_known.py holds the
device to this model bit for bit."""
from fractions import Fraction

import numpy as np
import pytest

import pyoracle_field
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN, capture, carve, check_enable, known_field, segments, walk
from densesurfelmapping_b200.elements import SEED_DTYPE

EPS = Fraction(1, 10 ** 9)


def interval(wa, wb, box_lo, box_hi, half_open=False):
    """The parameters t in [0, 1] at which wa + t (wb - wa) lies in the box (exact), or None.  half_open: a voxel
    [i, i + 1) on an axis the segment does not move along (a segment in a face belongs to the voxel above it)."""
    lo, hi = Fraction(0), Fraction(1)
    for k in range(3):
        a, d = wa[k], wb[k] - wa[k]
        if d == 0:
            if not (box_lo[k] <= a < box_hi[k] if half_open else box_lo[k] <= a <= box_hi[k]):
                return None
            continue
        t0, t1 = (box_lo[k] - a) / d, (box_hi[k] - a) / d
        lo, hi = max(lo, min(t0, t1)), min(hi, max(t0, t1))
    return (lo, hi) if lo <= hi else None


def exact_check(a, b):
    """One segment in voxel units (voxel edge 1): every voxel it crosses for more than EPS is visited; every visited
    voxel lies within EPS of it."""
    r, vox, _ = walk(np.array([a]), np.array([b]), 1.0)
    visited = {tuple(int(c) for c in q) for q in vox}
    assert len(visited) == len(vox), "a voxel was visited twice"
    wa, wb = [Fraction(float(x)) for x in a], [Fraction(float(x)) for x in b]
    length2 = sum((q - p) ** 2 for p, q in zip(wa, wb))
    for q in visited:
        assert interval(wa, wb, [c - EPS for c in q], [c + 1 + EPS for c in q]) is not None, f"{q} is off the segment {a} -> {b}"
    lo = [int(np.floor(min(x, y))) - 1 for x, y in zip(a, b)]
    hi = [int(np.floor(max(x, y))) + 1 for x, y in zip(a, b)]
    for x in range(lo[0], hi[0] + 1):
        for y in range(lo[1], hi[1] + 1):
            for z in range(lo[2], hi[2] + 1):
                iv = interval(wa, wb, [x, y, z], [x + 1, y + 1, z + 1], half_open=True)
                if iv is not None and (iv[1] - iv[0]) ** 2 * length2 > EPS * EPS:
                    assert (x, y, z) in visited, f"({x}, {y}, {z}) is crossed by {a} -> {b} and not visited"


def test_walk_against_exact_geometry():
    rng = np.random.default_rng(7)
    for _ in range(300):
        a, b = rng.uniform(-6, 6, 3), rng.uniform(-6, 6, 3)
        exact_check(a, b)
    for _ in range(100):   # short segments, and ends on integer planes
        a = rng.uniform(-3, 3, 3)
        exact_check(a, a + rng.uniform(-0.7, 0.7, 3))
        exact_check(np.round(a), np.round(a) + rng.integers(-3, 4, 3))


def visits(a, b, voxel=1.0):
    return [tuple(int(c) for c in q) for q in walk(np.array([a], float), np.array([b], float), voxel)[1]]


def test_axis_aligned_rays_and_the_tie_rule():
    assert visits((0.5, 0.5, 0.5), (4.5, 0.5, 0.5)) == [(x, 0, 0) for x in range(5)]
    assert visits((0.5, 3.5, 0.5), (0.5, 0.5, 0.5)) == [(0, y, 0) for y in (3, 2, 1, 0)]
    # exactly through corners: equal tM on every axis, x first, then y, then z
    assert visits((0.5, 0.5, 0.5), (2.5, 2.5, 2.5)) == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (1, 1, 1), (2, 1, 1), (2, 2, 1), (2, 2, 2)]
    # exactly along an edge (y = 1): the walk stays in the voxels at and above it
    assert visits((0.5, 1.0, 0.5), (3.5, 1.0, 0.5)) == [(x, 1, 0) for x in range(4)]
    # through an edge of two axes: the tie takes x before y
    assert visits((0.5, 0.5, 0.2), (1.5, 1.5, 0.2)) == [(0, 0, 0), (1, 0, 0), (1, 1, 0)]


def test_negative_coordinates():
    assert visits((-0.5, -0.5, -0.5), (-3.5, -0.5, -0.5)) == [(x, -1, -1) for x in (-1, -2, -3, -4)]
    assert visits((0.25, -0.25, 0.5), (-1.25, 0.75, 0.5)) == [(0, -1, 0), (-1, -1, 0), (-1, 0, 0), (-2, 0, 0)]
    assert visits((-0.1, -0.1, -0.1), (0.1, 0.1, 0.1), 0.5) == [(-1, -1, -1), (0, -1, -1), (0, 0, -1), (0, 0, 0)]


def pose(t=(0, 0, 0), R=np.eye(3)):
    P = np.zeros((3, 4))
    P[:, :3], P[:, 3] = R, t
    return P.reshape(12)


def run(views, voxel=1.0, shape=(8, 8, 8), center=(4, 4, 4), points=(), max_range=100.0):
    return known_field(np.asarray(points, np.float32).reshape(-1, 3), voxel, shape, center, views, max_range)


def test_a_ray_inside_one_voxel_carves_nothing():
    dist, _, n_occ, state, n_free = run([(np.array([[0.1, 0.2, 0.0]], np.float32), pose((2.5, 2.5, 2.5)))])
    assert n_free == 0 and n_occ == 0 and (state == UNKNOWN).all() and (dist == 0).all()


def test_the_end_voxel_holds_the_surface_unless_the_ray_was_truncated():
    ray = np.array([[3.0, 0.0, 0.0]], np.float32)   # from (1.5, 2.5, 2.5) to (4.5, 2.5, 2.5)
    _, _, _, state, n_free = run([(ray, pose((1.5, 2.5, 2.5)))])
    assert n_free == 3 and state[2, 2, 1:4].tolist() == [FREE] * 3 and state[2, 2, 4] == UNKNOWN
    _, _, _, state, n_free = run([(ray, pose((1.5, 2.5, 2.5)))], max_range=2.0)   # cut at (3.5, 2.5, 2.5)
    assert n_free == 3 and state[2, 2, 1:4].tolist() == [FREE] * 3 and state[2, 2, 4] == UNKNOWN
    a, b, trunc = segments(ray, pose((1.5, 2.5, 2.5)), 2.0)
    assert trunc.tolist() == [True] and b.tolist() == [[3.5, 2.5, 2.5]]
    _, _, _, state, n_free = run([(ray, pose((1.5, 2.5, 2.5)))], max_range=2.5)  # cut at (4.0, ...): voxel 4 carved
    assert n_free == 4 and state[2, 2, 1:5].tolist() == [FREE] * 4


def test_cameras_and_rays_outside_the_grid():
    # the grid covers [0, 8)^3; a camera at x = -5.5 whose ray crosses the grid along x carves the row up to its end
    ray = np.array([[10.0, 0.0, 0.0]], np.float32)
    _, _, _, state, n_free = run([(ray, pose((-5.5, 3.5, 3.5)))])
    assert n_free == 4 and state[3, 3, :4].tolist() == [FREE] * 4 and state[3, 3, 4] == UNKNOWN
    # rays that never enter it
    away = np.array([[-3.0, 0.0, 0.0], [0.0, 5.0, 0.0], [0.0, 0.0, -9.0]], np.float32)
    _, _, _, state, n_free = run([(away, pose((-5.5, 3.5, 3.5))), (away, pose((20.0, 20.0, 20.0)))])
    assert n_free == 0
    # a rotated camera: R maps the camera's z onto the world's -y
    R = np.array([[1.0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])
    _, _, _, state, n_free = run([(np.array([[0.0, 0.0, 6.0]], np.float32), pose((1.5, 7.5, 1.5), R))])
    assert n_free == 6 and state[1, 2:8, 1].tolist() == [FREE] * 6


def test_occupied_beats_free_and_n_views_zero_gives_zero():
    pts = [(4.5, 3.5, 3.5)]
    ray = np.array([[14.0, 0.0, 0.0]], np.float32)   # through the occupied voxel, to x = 8.5 outside the grid
    dist, _, n_occ, state, n_free = run([(ray, pose((-5.5, 3.5, 3.5)))], points=pts)
    assert n_occ == 1 and state[3, 3, 4] == OCCUPIED and state[3, 3, :4].tolist() == [FREE] * 4 and state[3, 3, 5:].tolist() == [FREE] * 3
    assert n_free == 7
    dist, _, n_occ, state, n_free = run([], points=pts)
    assert n_occ == 1 and n_free == 0 and (dist == 0).all() and dist.dtype == np.float32
    dist, _, n_occ, state, n_free = run([])
    assert n_occ == 0 and (dist == 0).all()


def rows_views(voxel, shape, center):
    """One view per x-row, from outside the grid through the whole row: every voxel is visited and none is an end."""
    nx, ny, nz = shape
    o = pyoracle_field.origin(center, voxel, shape)
    v = float(np.float32(voxel))
    ray = np.array([[(nx + 4) * v, 0.0, 0.0]], np.float32)
    return [(ray, pose(((o[0] - 1.5) * v, (o[1] + y + 0.5) * v, (o[2] + z + 0.5) * v))) for z in range(nz) for y in range(ny)]


@pytest.mark.parametrize("with_points", [False, True])
def test_every_voxel_free_equals_the_plain_field(with_points):
    voxel, shape, center = 0.25, (9, 6, 5), (0.3, -0.2, 1.1)
    rng = np.random.default_rng(3)
    pts = rng.uniform(-1.5, 1.5, (12, 3)).astype(np.float32) + np.float32(center) if with_points else np.zeros((0, 3), np.float32)
    dist, origin, n_occ, state, n_free = known_field(pts, voxel, shape, center, rows_views(voxel, shape, center), 100.0)
    plain = pyoracle_field.field(pts, voxel, shape, center)
    assert (state != UNKNOWN).all() and n_free + n_occ == state.size
    assert n_occ == plain[2] and origin.tolist() == plain[1].tolist()
    assert dist.tobytes() == plain[0].tobytes()
    if not with_points:
        assert np.isposinf(dist).all()


def test_known_never_exceeds_plain_on_random_scenes():
    rng = np.random.default_rng(11)
    for trial in range(12):
        voxel = float(rng.choice([0.1, 0.25, 0.5]))
        shape = tuple(int(n) for n in rng.integers(4, 24, 3))
        center = rng.uniform(-3, 3, 3)
        pts = (center + rng.normal(0, 1.5, (60, 3))).astype(np.float32)
        views = []
        for _ in range(int(rng.integers(0, 5))):
            q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
            t = center + rng.uniform(-2, 2, 3)
            views.append((rng.uniform(-3, 3, (200, 3)).astype(np.float32), pose(t, q)))
        dist, origin, n_occ, state, n_free = known_field(pts, voxel, shape, center, views, float(rng.choice([1.0, 2.0, 100.0])))
        plain = pyoracle_field.field(pts, voxel, shape, center)
        assert n_occ == plain[2] and origin.tolist() == plain[1].tolist()
        assert (dist <= plain[0]).all(), trial
        assert ((state == OCCUPIED) == (plain[0] == 0)).all()
        assert n_free == int((state == FREE).sum())


def test_capture_predicate():
    s = np.zeros(6, SEED_DTYPE)
    s["posi_x"], s["posi_y"], s["posi_z"] = np.arange(6), 1.0, 2.0
    s["mean_depth"] = [1.0, 0.0, -1.0, np.nan, 2.0, 3.0]
    s["posi_y"][4] = np.nan
    s["posi_z"][5] = np.inf
    assert capture(s).tolist() == [[0.0, 1.0, 2.0]]
    s["mean_depth"] = 1.0
    s["posi_y"][4], s["posi_z"][5] = 1.0, 2.0
    assert capture(s)[:, 0].tolist() == [0, 1, 2, 3, 4, 5]   # seed index order


def test_refused_requests():
    for bad in [(0, 10.0), (65537, 10.0), (4, 0.0), (4, -1.0), (4, float("nan")), (4, float("inf")), (4, 1024 * 0.1 * 1.001)]:
        with pytest.raises(ValueError):
            check_enable(bad[0], bad[1], 0.1)
    check_enable(1, 1024 * 0.125, 0.125)
    check_enable(65536, 1e-3, 0.1)
    ray = np.array([[1.0, 0, 0]], np.float32)
    for k in range(12):
        p = pose((1, 1, 1))
        p[k] = np.nan
        with pytest.raises(ValueError):
            run([(ray, p)])
    with pytest.raises(ValueError):
        run([], center=(0.5 * 2 ** 24, 0, 0), voxel=0.5)


def test_carve_writes_only_over_unknown():
    state = np.array([[[OCCUPIED, UNKNOWN, OCCUPIED, UNKNOWN]]], np.uint8)
    carve(state, [(np.array([[10.0, 0, 0]], np.float32), pose((-0.5, 0.5, 0.5)))], 1.0, np.array([0, 0, 0]), 100.0)
    assert state.tolist() == [[[OCCUPIED, FREE, OCCUPIED, FREE]]]
