"""oracle/pyoracle_field, the definition of dsm_field_enqueue's distance field, against a brute-force minimum over the
occupied voxels, and on hand-made points at the edges of the definition: voxel boundaries on both sides of zero, the
faces of the grid, non-finite and huge coordinates, empty and single-voxel grids, thin and odd shapes.
tests/test_gpu_field.py holds the device to this model bit for bit."""
import numpy as np
import pytest

import pyoracle_field
from pyoracle_field import field


def brute(points, voxel, shape, center):
    """The definition again, voxel by voxel: an independent restatement of occupancy and distance."""
    nx, ny, nz = shape
    v = np.float32(voxel)
    o = [int(np.floor(np.float64(c) / np.float64(v))) - n // 2 for c, n in zip(center, shape)]
    occ = set()
    for p in np.asarray(points, np.float32).reshape(-1, 3):
        q = []
        for k in range(3):
            with np.errstate(invalid="ignore", over="ignore"):
                qk = np.floor(np.float32(p[k]) / v)
            if not (qk >= np.float32(o[k]) and qk < np.float32(o[k] + shape[k])):
                break
            q.append(int(qk) - o[k])
        else:
            occ.add(tuple(q))
    dist = np.full((nz, ny, nx), np.inf, np.float32)
    if occ:
        occ_a = np.array(sorted(occ), np.int64)
        zz, yy, xx = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
        grid = np.stack([xx, yy, zz], -1).reshape(-1, 1, 3)
        d2 = ((grid - occ_a[None]) ** 2).sum(-1).min(1).reshape(nz, ny, nx)
        dist = np.sqrt(d2.astype(np.float32)) * v
    return dist, np.array(o, np.int32), len(occ)


def same(a, b):
    assert a[0].dtype == np.float32 and a[0].shape == b[0].shape
    assert a[0].tobytes() == b[0].tobytes(), "distances differ"
    assert a[1].tolist() == b[1].tolist() and a[2] == b[2]


@pytest.mark.parametrize("seed", range(40))
def test_random_grids_equal_the_brute_force_minimum(seed):
    rng = np.random.default_rng(seed)
    shape = tuple(int(s) for s in rng.integers(1, 13, 3))
    voxel = float(rng.choice([0.1, 0.125, 0.3, 1.0, 0.07]))
    center = rng.normal(scale=3.0, size=3)
    n = int(rng.integers(0, 30))
    span = np.array(shape) * voxel
    pts = center + (rng.random((n, 3)) - 0.5) * span * 1.4
    got = field(pts.astype(np.float32), voxel, shape, center)
    same(got, brute(pts, voxel, shape, center))
    assert got[2] <= n


def test_boundaries_use_floor_not_truncation():
    v = 0.25
    shape = (8, 1, 1)
    o = pyoracle_field.origin([0.0, 0.0, 0.0], v, shape)
    assert o.tolist() == [-4, 0, 0]
    for x, want in [(-0.25, 3), (-1.0, 0), (0.0, 4), (0.75, 7), (-0.2, 3), (0.2, 4)]:
        d, org, n = field(np.array([[x, 0.0, 0.0]], np.float32), v, shape, [0.0, 0.0, 0.0])
        assert n == 1 and d[0, 0, want] == 0.0, x
    # one ulp below a boundary falls into the voxel below it
    below = np.nextafter(np.float32(-0.5), np.float32(-1.0))
    d, _, _ = field(np.array([[below, 0, 0]], np.float32), v, shape, [0.0, 0.0, 0.0])
    assert d[0, 0, 1] == 0.0 and d[0, 0, 2] == np.float32(v)
    below = np.nextafter(np.float32(0.5), np.float32(0.0))
    d, _, _ = field(np.array([[below, 0, 0]], np.float32), v, shape, [0.0, 0.0, 0.0])
    assert d[0, 0, 5] == 0.0 and d[0, 0, 6] == np.float32(v)


@pytest.mark.parametrize("axis", range(3))
def test_faces(axis):
    v, shape, c = 0.5, (4, 5, 6), np.array([0.3, -0.7, 1.1])
    o = pyoracle_field.origin(c, v, shape)
    lo, hi = o[axis] * v, (o[axis] + shape[axis]) * v
    base = (o + np.array(shape) // 2) * v + v / 2
    for x, inside in [(lo, True), (lo - 1e-3, False), (hi - 1e-3, True), (hi, False)]:
        p = base.copy()
        p[axis] = x
        got = field(p[None].astype(np.float32), v, shape, c)
        assert got[2] == int(inside), (axis, x)
        same(got, brute(p[None], v, shape, c))


def test_non_finite_and_huge_coordinates_mark_nothing():
    pts = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e30, 0, 0], [-1e30, 0, 0], [0, 0, 1e30]], np.float32)
    d, _, n = field(pts, 0.1, (5, 5, 5), [0.0, 0.0, 0.0])
    assert n == 0 and np.isposinf(d).all()
    d, _, n = field(np.vstack([pts, [[0.0, 0.0, 0.0]]]).astype(np.float32), 0.1, (5, 5, 5), [0.0, 0.0, 0.0])
    assert n == 1 and d[2, 2, 2] == 0.0


def test_empty_grid():
    d, o, n = field(np.zeros((0, 3), np.float32), 0.2, (3, 4, 5), [10.0, -3.0, 0.5])
    assert n == 0 and d.shape == (5, 4, 3) and np.isposinf(d).all() and d.dtype == np.float32


def test_single_occupied_voxel_closed_form():
    v, shape = np.float32(0.3), (7, 6, 5)
    c = [-2.0, 4.0, -0.1]
    o = pyoracle_field.origin(c, v, shape)
    cell = np.array([2, 4, 1])
    p = ((o + cell).astype(np.float64) + 0.5) * float(v)
    d, _, n = field(p[None].astype(np.float32), v, shape, c)
    assert n == 1
    zz, yy, xx = np.meshgrid(np.arange(5), np.arange(6), np.arange(7), indexing="ij")
    d2 = (xx - cell[0]) ** 2 + (yy - cell[1]) ** 2 + (zz - cell[2]) ** 2
    assert d.tobytes() == (np.sqrt(d2.astype(np.float32)) * v).tobytes()


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 9, 1), (11, 1, 3), (1, 1, 12), (5, 7, 9)])
def test_thin_and_odd_shapes_with_negative_centres(shape):
    rng = np.random.default_rng(sum(shape))
    c = np.array([-3.3, -0.01, -7.9])
    pts = c + rng.normal(scale=0.4, size=(20, 3))
    same(field(pts.astype(np.float32), 0.2, shape, c), brute(pts, 0.2, shape, c))


def test_origin_bound():
    v = 1.0
    assert pyoracle_field.origin([2.0 ** 24 - 10, 0, 0], v, (8, 1, 1)) is not None
    assert pyoracle_field.origin([2.0 ** 24, 0, 0], v, (8, 1, 1)) is None      # o + n above 2^24
    assert pyoracle_field.origin([-(2.0 ** 24) + 3, 0, 0], v, (8, 1, 1)) is None  # o below -2^24
    assert pyoracle_field.origin([1e300, 0, 0], v, (8, 1, 1)) is None
    with pytest.raises(ValueError):
        field(np.zeros((0, 3), np.float32), v, (8, 1, 1), [1e300, 0, 0])
