"""The exact distance transform of csrc/dsm_field.cu at the grid's limits: lines of up to 1024 voxels, the packed envelope
word, the opt-in shared memory of lines above 384 voxels, and points on voxel faces.

Every comparison is bit for bit.  The known path (dsm_debug_field_load_state) equals oracle/pyoracle_field_known on an
axis sweep of 1 to 1024 voxels with uniform grids, single sites at the corners and the centre, the ends of every long
line, random sites and far origins, and on the three wide planes of 1024 x 1024 voxels with the crafted patterns of
tests/edt_patterns.py, whose branches tests/test_field_edt_model.py proves on the host.  The plain path
(dsm_field_enqueue) equals oracle/pyoracle_field on obstacle points at fp32 multiples of the voxel edge and their ulp
neighbours, non-finite and huge coordinates, and pool surfels on both sides of min_update_times.  The largest grid the
API accepts, 1024^3 (a 4 GiB distance grid), is queried at its corners and at thousands of points against the closed
form."""
import numpy as np
import pytest

import edt_patterns as P
import pyoracle_field
import pyoracle_field_query
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import FREE, OCCUPIED, SMALL_CAM, UNKNOWN, small_ctx
from resident_map import assert_field, load_known

pytestmark = pytest.mark.gpu

LIM = 1 << 24
LENGTHS = [1, 2, 31, 32, 33, 320, 384, 385, 512, 1023, 1024]
SWEEP = [s for n in LENGTHS for s in ((n, 3, 5), (5, n, 3), (3, 5, n))] + [(33, 385, 1023)]


def sid(s):
    return "x".join(map(str, s))


def known_ctx(shape, voxel=0.2):
    """A context whose field has grid `shape` (nx, ny, nz) and views enabled, as the frontier loaders make."""
    return small_ctx(shape, voxel)


def states(sites, rng):
    """Free everywhere but the sites, which are unknown or occupied at random."""
    st = np.full(sites.shape, FREE, np.uint8)
    st[sites] = rng.choice([UNKNOWN, OCCUPIED], size=int(sites.sum())).astype(np.uint8)
    return st


def origins(shape):
    nx, ny, nz = shape
    return [(0, 0, 0), (-7, 3, -1024), (1000, -5, 12), (-LIM, LIM - ny, 5), (LIM - nx, -LIM, -LIM)]


# ---- the known path ----
@pytest.mark.parametrize("shape", SWEEP, ids=sid)
def test_axis_sweep(shape):
    rng = np.random.default_rng(sum(shape) * 31 + shape[0])
    voxel = 0.2
    grids = [np.full(shape[::-1], s, np.uint8) for s in (FREE, UNKNOWN, OCCUPIED)]
    grids += [states(m, rng) for m in P.corners_and_centre(shape)]
    grids.append(states(P.line_ends(shape), rng))
    grids += [states(P.random_sites(shape, d, rng), rng) for d in (1e-4, 1e-2, 0.3)]
    org = origins(shape)
    ctx = known_ctx(shape, voxel)
    for k, st in enumerate(grids):
        dist = load_known(ctx, st, org[k % len(org)], voxel, f"{shape} grid {k}")
        if k == 0:
            assert np.isposinf(dist).all()
        elif k < 3:
            assert (dist == 0).all()
    ctx.close()


@pytest.mark.parametrize("shape", P.WIDE, ids=sid)
def test_wide_planes(shape):
    """Lines of 1024 voxels along both long axes with the crafted patterns: a full envelope, pops to empty and to a
    non-empty envelope, drops, exact separators, a tie at t_top, and the largest packed f."""
    rng = np.random.default_rng(sum(shape))
    voxel = 0.1
    ctx = known_ctx(shape, voxel)
    for name, fn in P.PLANES.items():
        st = states(P.grid(fn(), shape), rng)
        dist = load_known(ctx, st, (-3, 11, -512), voxel, f"{shape} {name}")
        if name == "corner":
            far = 2 * (P.L - 1) ** 2
            assert dist.max() == np.sqrt(np.float32(far)) * np.float32(voxel)
    ctx.close()


# ---- the plain path: obstacle points ----
VOXELS = [0.1, 0.3, 0.07, 0.125]
PLAIN = [(48, 40, 36), (1024, 3, 5), (5, 1024, 3), (3, 5, 1024)]


def surfels(points, update_times, last_update=0):
    s = np.zeros(len(points), SURFEL_DTYPE)
    p = np.asarray(points, np.float32).reshape(-1, 3)
    s["px"], s["py"], s["pz"] = p[:, 0], p[:, 1], p[:, 2]
    s["update_times"] = update_times
    s["last_update"] = last_update
    return s


def plain_ctx(shape, voxel):
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 14)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.inactive_reserve(1 << 14)
    ctx.field_enable(voxel, *shape)
    return ctx


def centre_for(o, shape, voxel):
    """A request centre whose origin is o: the middle of voxel o + n // 2."""
    v = np.float64(np.float32(voxel))
    return [(o[k] + shape[k] // 2 + 0.5) * v for k in range(3)]


def plain_equals_oracle(ctx, shape, voxel, o, pool, store, m, what):
    """pool: (points, update_times); store: points, one segment of keyframe 3.  Returns (dist, origin, n_occupied)."""
    ctx.pool_upload(surfels(pool[0], pool[1]))
    ctx.inactive_load(surfels(store, 1, 3), [[3, 0, len(store)]] if len(store) else np.zeros((0, 3), np.int32))
    c = centre_for(o, shape, voxel)
    ctx.field_enqueue(c, m)
    got = ctx.field_wait()
    counted = np.concatenate([np.asarray(pool[0], np.float32).reshape(-1, 3)[np.asarray(pool[1]) >= m],
                              np.asarray(store, np.float32).reshape(-1, 3)])
    want = pyoracle_field.field(counted, voxel, shape, c)
    assert want[1].tolist() == list(o), what
    assert_field(got, want, what)
    return got


def face_points(shape, o, voxel, axis):
    """Along `axis`, for every k from o - 1 to o + n + 1 (the lo face k = o, the hi face k = o + n outside, one ulp below
    it inside): float32(k) * v and its two ulp neighbours, each at the centre of its own line of the other two axes, so
    that a point placed one voxel off changes the field."""
    v = np.float32(voxel)
    others = [k for k in range(3) if k != axis]
    n1, n2 = shape[others[0]], shape[others[1]]
    pts = []
    j = 0
    for k in range(o[axis] - 1, o[axis] + shape[axis] + 2):
        p = np.float32(k) * v
        for q in (np.nextafter(p, np.float32(-np.inf)), p, np.nextafter(p, np.float32(np.inf))):
            line = (j * 7) % (n1 * n2)
            pt = np.zeros(3, np.float32)
            pt[axis] = q
            pt[others[0]] = np.float32((o[others[0]] + line % n1 + 0.5) * np.float64(v))
            pt[others[1]] = np.float32((o[others[1]] + line // n1 + 0.5) * np.float64(v))
            pts.append(pt)
            j += 1
    return np.array(pts, np.float32)


@pytest.mark.parametrize("shape", PLAIN, ids=sid)
@pytest.mark.parametrize("voxel", VOXELS)
def test_points_on_voxel_faces(voxel, shape):
    """Each axis in turn, at an origin across zero and at far ones of both signs; half of the points in the pool (at
    min_update_times), half in the store."""
    ctx = plain_ctx(shape, voxel)
    for o in [tuple(-(n // 2) - 1 for n in shape), (-5000, 3001, -77), (4093, -9000, 250)]:
        for axis in range(3):
            pts = face_points(shape, o, voxel, axis)
            got = plain_equals_oracle(ctx, shape, voxel, o, (pts[0::2], np.full(len(pts[0::2]), 5)), pts[1::2], 5,
                                      f"{shape} v={voxel} o={o} axis {axis}")
            assert 0 < got[2] < len(pts)
    ctx.close()


@pytest.mark.parametrize("shape", PLAIN, ids=sid)
def test_non_finite_and_huge_coordinates(shape):
    voxel = 0.1
    o = tuple(-(n // 2) for n in shape)
    mid = np.array([(o[k] + shape[k] // 2 + 0.5) * np.float64(np.float32(voxel)) for k in range(3)], np.float32)
    bad = []
    for axis in range(3):
        for x in (np.nan, np.inf, -np.inf, 1e30, -1e30):
            p = mid.copy()
            p[axis] = x
            bad.append(p)
    bad = np.array(bad, np.float32)
    ctx = plain_ctx(shape, voxel)
    got = plain_equals_oracle(ctx, shape, voxel, o, (bad, np.full(len(bad), 5)), bad, 5, f"{shape} non-finite only")
    assert got[2] == 0 and np.isposinf(got[0]).all()
    one = np.vstack([bad, mid[None]])
    got = plain_equals_oracle(ctx, shape, voxel, o, (one, np.full(len(one), 5)), bad, 5, f"{shape} and one point")
    assert got[2] == 1
    ctx.close()


@pytest.mark.parametrize("shape", PLAIN, ids=sid)
@pytest.mark.parametrize("m", [1, 5])
def test_pool_surfels_on_both_sides_of_min_update_times(m, shape):
    voxel = 0.125
    rng = np.random.default_rng(m * 1000 + sum(shape))
    o = tuple(-(n // 2) for n in shape)
    v = np.float64(np.float32(voxel))
    lo, hi = np.array(o) * v, (np.array(o) + np.array(shape)) * v
    pool = (lo + rng.random((400, 3)) * (hi - lo)).astype(np.float32)
    ut = rng.choice([m - 1, m], size=len(pool))
    store = (lo + rng.random((20, 3)) * (hi - lo)).astype(np.float32)
    ctx = plain_ctx(shape, voxel)
    got = plain_equals_oracle(ctx, shape, voxel, o, (pool, ut), store, m, f"{shape} m={m}")
    assert got[2] > 0
    got = plain_equals_oracle(ctx, shape, voxel, o, (pool, ut), np.zeros((0, 3), np.float32), m, f"{shape} m={m}, pool only")
    assert got[2] > 0
    ctx.close()


# ---- the largest grid ----
def test_largest_grid_against_the_closed_form():
    """1024^3 at v = 1/8, resident: a stored surfel in voxel (0,0,0) alone (min_update_times 5), then with a pool
    surfel of 3 updates elsewhere (min_update_times 1).  Queries at the eight corner centres (the far one at
    d2 = 3 * 1023^2), at random voxel centres and at dyadic points, against pyoracle_field_query.sample on the 2x2x2
    sub-grid of each point's corners, built from the closed form.  At v = 1/8 on dyadic points every fp64 addressing
    step is exact, so the sub-grid gives the same corners and fractions as the whole grid."""
    n, voxel = 1024, 0.125
    v = np.float64(voxel)
    o = np.array([-512, -512, -512])
    centre = (0.0625, 0.0625, 0.0625)
    rng = np.random.default_rng(1024)
    corners = np.array([(x, y, z) for z in (0, n - 1) for y in (0, n - 1) for x in (0, n - 1)], np.float64)
    u = np.vstack([corners, rng.integers(0, n, (2000, 3)).astype(np.float64),
                   rng.integers(0, 8 * (n - 1) + 1, (2000, 3)) / 8.0,
                   [[n - 1, 0.125, 511.5], [0.0, n - 1.125, n - 1]]])
    pts = (o + 0.5 + u) * v
    stored = ((o + 0.5) * v)[None].astype(np.float32)
    other = np.array([700, 300, 900])
    pool = ((o + other + 0.5) * v)[None].astype(np.float32)
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(surfels(pool, 3))
    ctx.inactive_reserve(16)
    ctx.inactive_load(surfels(stored, 1, 3), [[3, 0, 1]])
    ctx.field_enable(voxel, n, n, n)
    ctx.field_query_enable(len(pts), 0, 0)
    for m, sites in [(5, [np.zeros(3, np.int64)]), (1, [np.zeros(3, np.int64), other])]:
        ctx.field_enqueue(centre, m, host_copy=False)
        dist, origin, n_occ = ctx.field_wait()
        assert dist is None and origin.tolist() == o.tolist() and n_occ == len(sites)
        ctx.field_query_enqueue(points=pts)
        got, _ = ctx.field_query_wait()
        want = np.zeros(len(pts), pyoracle_field_query.SAMPLE_DTYPE)
        for q in range(len(pts)):
            i = np.minimum(np.floor(u[q]), n - 2).astype(np.int64)
            c = np.indices((2, 2, 2)).reshape(3, -1).T[:, ::-1] + i      # (x, y, z) of the corners, z slowest
            d2 = np.min([((c - s) ** 2).sum(1) for s in sites], axis=0)
            sub = (np.sqrt(d2.astype(np.float32)) * np.float32(voxel)).reshape(2, 2, 2)
            want[q] = pyoracle_field_query.sample(sub, o + i, voxel, pts[q][None])[0]
        bad = np.flatnonzero((got.view(np.uint32).reshape(-1, 4) != want.view(np.uint32).reshape(-1, 4)).any(1))
        assert got.tobytes() == want.tobytes(), f"m={m}: {len(bad)} samples differ, first {bad[:4]}"
        if m == 5:
            far = np.float32(np.sqrt(np.float32(3 * (n - 1) ** 2)) * np.float32(voxel))
            assert got["dist"][7] == far and got["dist"][0] == 0.0
    ctx.close()
