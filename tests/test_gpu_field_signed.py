"""dsm_field_signed_enable, dsm_field_signed and dsm_field_query_enqueue_signed: the signed distance field.

Every signed grid equals oracle/pyoracle_field_signed bit for bit: the windowed drive's plain and known fields (chunks
of 1 and 4 frames, loop-closure warps between calls, host copy and resident), crafted state grids through
dsm_debug_field_load_state with the states of tests/edt_patterns.py swapped 2 <-> 0 so that the complement transform
meets each envelope branch, at every line length of tests/test_gpu_field_edt.py up to 1024 voxels, and the +-INFINITY
rules.  Signed queries equal the oracle's, and on a resident field match the host copy of a twin at voxel centres.  A
twin context without the signed grid gives byte-identical distances, states, frontiers, reach, queries, map and
published clouds.  The rejected-frame and error contracts, and dsm::SurfelMapNode (tests/cpp/field_signed_main.cpp)."""
import filecmp

import numpy as np
import pytest

import edt_patterns as P
import pyoracle_field_known
import pyoracle_field_query as fq
import pyoracle_field_signed as fs
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from known_space import FREE, MAX_RANGE, NODE_FIELD, OCCUPIED, UNKNOWN, Views, small_ctx
from node_drive import node_script, run_driver
from resident_map import SHAPES, STORE, T, camera, field_points, map_state, new_ctx, simple_lists, warp, windowed, xyz

pytestmark = pytest.mark.gpu

LENGTHS = [1, 2, 31, 32, 33, 320, 384, 385, 512, 1023, 1024]
SWEEP = [s for n in LENGTHS for s in ((n, 3, 5), (5, n, 3), (3, 5, n))] + [(33, 385, 1023)]
CAPS = (4096, 64, 512)


def sid(s):
    return "x".join(map(str, s))


def differ(a, b):
    return int((np.asarray(a).view(np.uint32) != np.asarray(b).view(np.uint32)).sum())


def centre_points(rng, origin, voxel, shape, n=2000):
    """Voxel centres (none on an axis's last voxel, where the interpolation's fraction is 1), random points in and around
    the box, and a non-finite one."""
    v = float(np.float32(voxel))
    o, n3 = np.asarray(origin, np.float64), np.array(shape, np.float64)
    cells = rng.integers(0, np.maximum(np.array(shape) - 1, 1), (n, 3))
    rnd = (o - 1 + rng.random((n, 3)) * (n3 + 2)) * v
    return np.concatenate([(cells + o + 0.5) * v, rnd, [[np.nan, 0, 0]]]), cells


def trajectories(rng, origin, voxel, shape, n=32):
    v = float(np.float32(voxel))
    o, n3 = np.asarray(origin, np.float64), np.array(shape, np.float64)
    k = rng.integers(1, 9, n)
    ofs = np.concatenate([[0], np.cumsum(k)]).astype(np.int32)
    wp = (o - 1 + rng.random((int(ofs[-1]), 3)) * (n3 + 2)) * v
    return wp, ofs


def signed_query_equals_oracle(ctx, sdist, origin, voxel, shape, rng, what):
    pts, _ = centre_points(rng, origin, voxel, shape, 1000)
    wp, ofs = trajectories(rng, origin, voxel, shape)
    step, radius = float(np.float32(voxel)) / 2, 2 * float(np.float32(voxel))
    ctx.field_query_enqueue(pts, wp, ofs, step, radius, signed=True)
    s, c = ctx.field_query_wait()
    ws = fs.sample(sdist, origin, voxel, pts)
    wc = fs.clearance(sdist, origin, voxel, wp, ofs, step, radius)
    assert s.tobytes() == ws.tobytes(), f"{what}: {differ(s.view(np.float32), ws.view(np.float32))} sample words differ"
    assert c.tobytes() == wc.tobytes(), f"{what}: clearance"
    return s, c


# ---- the windowed drive ----
@pytest.mark.parametrize("shape", SHAPES[:3], ids=sid)
@pytest.mark.parametrize("chunk", [1, 4])
def test_drive_fields_equal_the_oracle(chunk, shape):
    """After every windowed call one field, alternating plain and known, host copy and resident (every second pair),
    the voxel edge cycling through 0.125, 0.1 and 0.3 across the shapes; loop-closure warps every second call.  Host
    copies are held to the oracle's grid, resident fields through signed queries."""
    lists = simple_lists()
    voxel = {SHAPES[0]: 0.125, SHAPES[1]: 0.1, SHAPES[2]: 0.3}[shape]
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_signed_enable()
    ctx.field_query_enable(*CAPS)
    views = Views(ctx, 6)
    rng = np.random.default_rng(chunk * 7 + sum(shape))
    stored, negative = set(), 0
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        windowed(ctx, t0, t1, lists, want_counts=False)
        views.capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            ctx.pool_transform(warp(1))
            ctx.inactive_transform(max(stored), warp(2))
            views.warp(warp(1))
        known, host_copy = call % 2 == 1, call % 4 < 2
        c = camera(t1 - 1)
        what = f"frames {t0}-{t1 - 1} {'known' if known else 'plain'} {'host' if host_copy else 'resident'}"
        if known:
            slots, poses = views.request()
            ctx.field_enqueue_known(c, 5, slots, poses, host_copy=host_copy)
            dist, origin, n_occ = ctx.field_wait()
            want = pyoracle_field_known.known_field(field_points(ctx, 5), voxel, shape, c, views.oracle_views(slots), MAX_RANGE)
            wd, ws = fs.state_field(want[3], voxel)
        else:
            ctx.field_enqueue(c, 5, host_copy=host_copy)
            dist, origin, n_occ = ctx.field_wait()
            wd, ws, o, n = fs.field(field_points(ctx, 5), voxel, shape, c)
            want = (wd, o, n)
        assert origin.tolist() == want[1].tolist() and n_occ == want[2], what
        sdist = ctx.field_signed()
        if host_copy:
            assert dist.tobytes() == wd.tobytes(), f"{what}: dist"
            assert sdist.tobytes() == ws.tobytes(), f"{what}: {differ(sdist, ws)} signed voxels differ"
        else:
            assert dist is None and sdist is None
        signed_query_equals_oracle(ctx, ws, origin, voxel, shape, rng, what)
        negative += int((ws < 0).any())
    assert negative > 0 or shape == (1, 1, 1)
    ctx.close()


# ---- crafted grids ----
def known_ctx(shape, voxel=0.2):
    ctx = small_ctx(shape, voxel)
    ctx.field_signed_enable()
    return ctx


def swapped(sites, rng):
    """The complement of test_gpu_field_edt's states: free on the pattern's sites, unknown or occupied elsewhere, so
    that F is the pattern."""
    st = rng.choice([UNKNOWN, OCCUPIED], size=sites.shape).astype(np.uint8)
    st[sites] = FREE
    return st


def load_signed(ctx, state, origin, voxel, what):
    ctx.debug_field_load_state(np.ascontiguousarray(state, np.uint8), origin)
    dist, org, _ = ctx.field_wait()
    sdist = ctx.field_signed()
    wd, ws = fs.state_field(state, voxel)
    assert dist.tobytes() == wd.tobytes(), f"{what}: dist"
    assert sdist.tobytes() == ws.tobytes(), f"{what}: {differ(sdist, ws)} signed voxels differ"
    return sdist


@pytest.mark.parametrize("shape", SWEEP, ids=sid)
def test_axis_sweep(shape):
    rng = np.random.default_rng(sum(shape) * 13 + shape[1])
    voxel = 0.2
    ctx = known_ctx(shape, voxel)
    grids = [np.full(shape[::-1], s, np.uint8) for s in (FREE, UNKNOWN, OCCUPIED)]
    grids += [swapped(m, rng) for m in P.corners_and_centre(shape)]
    grids.append(swapped(P.line_ends(shape), rng))
    grids += [swapped(P.random_sites(shape, d, rng), rng) for d in (1e-4, 1e-2, 0.3)]
    for k, st in enumerate(grids):
        sdist = load_signed(ctx, st, (k * 3 - 7, 5, -1024), voxel, f"{shape} grid {k}")
        if k == 0:
            assert np.isposinf(sdist).all()
        elif k < 3:
            assert np.isneginf(sdist).all()
    ctx.close()


@pytest.mark.parametrize("shape", P.WIDE, ids=sid)
def test_wide_planes(shape):
    rng = np.random.default_rng(sum(shape) + 1)
    voxel = 0.1
    ctx = known_ctx(shape, voxel)
    for name, fn in P.PLANES.items():
        sdist = load_signed(ctx, swapped(P.grid(fn(), shape), rng), (-3, 11, -512), voxel, f"{shape} {name}")
        if name == "corner":
            assert sdist.min() == (np.float32(1) - np.sqrt(np.float32(2 * (P.L - 1) ** 2))) * np.float32(voxel)
    ctx.close()


def test_signed_queries_and_the_infinity_rules():
    """Queries on loaded grids: all free (+inf), all unknown (-inf), a half-free box whose gradient deep in the unknown
    half points to the free half, and random states."""
    shape, voxel = (40, 24, 16), 0.1
    ctx = known_ctx(shape, voxel)
    ctx.field_query_enable(*CAPS)
    rng = np.random.default_rng(3)
    o = (5, -3, 2)
    half = np.full(shape[::-1], UNKNOWN, np.uint8)
    half[:, :, :10] = FREE
    grids = {"free": np.full(shape[::-1], FREE, np.uint8), "unknown": np.full(shape[::-1], UNKNOWN, np.uint8), "half": half,
             "random": rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1], p=[0.3, 0.1, 0.6]).astype(np.uint8)}
    for name, st in grids.items():
        sdist = load_signed(ctx, st, o, voxel, name)
        s, c = signed_query_equals_oracle(ctx, sdist, np.array(o), voxel, shape, rng, name)
        inside = ~np.isnan(s["dist"])
        if name == "free":
            assert np.isposinf(s["dist"][inside]).all() and (s["gx"] == 0).all()
        if name == "unknown":
            assert np.isneginf(s["dist"][inside]).all() and (s["gx"] == 0).all() and np.isneginf(c["min_dist"]).all()
        if name == "half":
            p = (np.array([[30.2, 12.0, 8.0]]) + o + 0.5) * np.float64(np.float32(voxel))
            ctx.field_query_enqueue(p, signed=True)
            g, _ = ctx.field_query_wait()
            assert g["dist"][0] < -1.5 and g["gx"][0] < 0 and g["gy"][0] == 0 and g["gz"][0] == 0
            ctx.field_query_enqueue(p)
            u, _ = ctx.field_query_wait()
            assert u["dist"][0] == 0 and u["gx"][0] == 0
            assert (c["min_dist"] < 0).any()
    ctx.close()


def test_resident_queries_match_a_twins_host_copy():
    """At voxel centres a signed query returns the voxel's value: a resident request and a host-copy twin agree."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.125
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.field_signed_enable()
    a.field_query_enable(*CAPS)
    va, vb = Views(a, 4), Views(b, 4)
    for call, t0 in enumerate(range(0, 8, 2)):
        for c, v in ((a, va), (b, vb)):
            windowed(c, t0, t0 + 2, lists, want_counts=False)
            v.capture_call(call, t0, t0 + 2)
    rng = np.random.default_rng(11)
    for known in (False, True):
        cam = camera(7)
        if known:
            sl, po = va.request()
            a.field_enqueue_known(cam, 5, sl, po, host_copy=False)
            b.field_enqueue_known(cam, 5, *vb.request())
        else:
            a.field_enqueue(cam, 5, host_copy=False)
            b.field_enqueue(cam, 5)
        _, origin, _ = a.field_wait()
        b.field_wait()
        assert a.field_signed() is None
        host = b.field_signed()
        pts, cells = centre_points(rng, origin, voxel, shape, 3000)
        a.field_query_enqueue(pts[:len(cells)], signed=True)
        s, _ = a.field_query_wait()
        want = host[cells[:, 2], cells[:, 1], cells[:, 0]]
        assert s["dist"].tobytes() == want.tobytes(), f"known={known}: {differ(s['dist'], want)} centres differ"
        assert (want < 0).any() if known else True
    a.close()
    b.close()


# ---- nothing else changes ----
@pytest.mark.parametrize("chunk", [1, 4])
def test_signed_changes_nothing_else(chunk):
    """A context with the signed grid and a twin without it: byte-identical distances, states, frontiers, reach
    (with its cost grid), unsigned queries, map and published clouds."""
    lists = simple_lists()
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    shape, voxel = (64, 64, 32), 0.1
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.publish_enable()
        c.field_query_enable(*CAPS)
    va, vb = Views(a, 4), Views(b, 4)
    for c in (a, b):
        c.frontier_enable(256, 1 << 16)
        c.reach_enable(64, 1 << 16, 4096)
    a.field_signed_enable()
    rng = np.random.default_rng(chunk)
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c, v in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            v.capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            for c, v in ((a, va), (b, vb)):
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
                v.warp(warp(1))
        cam = camera(t1 - 1)
        what = f"after frames {t0}-{t1 - 1}"
        for c in (a, b):
            c.field_enqueue(cam, 5)
        fa, fb = a.field_wait(), b.field_wait()
        assert fa[0].tobytes() == fb[0].tobytes() and fa[2] == fb[2], f"{what}: plain field"
        for c, v in ((a, va), (b, vb)):
            c.field_enqueue_known(cam, 5, *v.request())
        fa, fb = a.field_wait(), b.field_wait()
        assert fa[0].tobytes() == fb[0].tobytes() and fa[2] == fb[2], f"{what}: known field"
        sa, sb = a.field_state(), b.field_state()
        assert sa[0].tobytes() == sb[0].tobytes() and sa[1] == sb[1], f"{what}: states"
        pts, _ = centre_points(rng, fa[1], voxel, shape, 500)
        wp, ofs = trajectories(rng, fa[1], voxel, shape)
        res = []
        for c in (a, b):
            c.frontier_enqueue(2)
            fr = c.frontier_wait()
            c.reach_enqueue(cam, 0.2, 1, None, True, True)
            re = c.reach_wait()
            c.field_query_enqueue(pts, wp, ofs, 0.05, 0.2)
            q = c.field_query_wait()
            c.publish_enqueue(5)
            pu = c.publish_wait()
            res.append([fr[0].tobytes(), fr[1].tobytes(), fr[2].tobytes(), re[0].tobytes(), re[1].tobytes(), re[2].tobytes(),
                        re[3].tobytes(), q[0].tobytes(), q[1].tobytes(), pu[0].tobytes(), pu[1].tobytes(), pu[2]])
        assert res[0] == res[1], f"{what}: {[k for k in range(len(res[0])) if res[0][k] != res[1][k]]} differ"
        assert map_state(a) == map_state(b), f"{what}: pool, store or table"
        with pytest.raises(capi.DsmError) as e:   # the twin has no signed grid
            b.field_signed()
        assert e.value.code == -7
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_signed():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    a = new_ctx(store=STORE)
    for t0 in range(0, first):
        windowed(a, t0, t0 + 1, lists, want_counts=False)
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    b.field_signed_enable()
    b.field_query_enable(*CAPS)
    for t0 in range(0, first + 2):
        windowed(b, t0, t0 + 1, lists, want_counts=False)
    c = camera(first - 1)
    b.field_enqueue(c, 1)
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6
    with pytest.raises(capi.DsmError) as e:
        b.field_signed()
    assert e.value.code == -6
    wd, ws, o, n = fs.field(field_points(a, 1), voxel, shape, c)
    assert e.value.signed.tobytes() == ws.tobytes() and n > 0
    pts, _ = centre_points(np.random.default_rng(1), o, voxel, shape, 200)
    b.field_query_enqueue(pts, signed=True)
    with pytest.raises(capi.DsmError) as e:
        b.field_query_wait()
    assert e.value.code == -6 and e.value.query[0].tobytes() == fs.sample(ws, o, voxel, pts).tobytes()
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    a.close()
    b.close()


def test_error_contract():
    lib = capi.load_library()
    C = (capi.ctypes.c_double * 3)
    P3 = capi.ctypes.c_void_p()
    pts = np.zeros((1, 3))

    def query(ctx):
        return lib.dsm_field_query_enqueue_signed(ctx.h, pts.ctypes.data, 1, None, None, 0, 1.0, 0.0)

    ctx = new_ctx(store=STORE)
    assert lib.dsm_field_signed_enable(None) == -1
    assert lib.dsm_field_signed(None, None) == -1
    assert lib.dsm_field_query_enqueue_signed(None, None, 0, None, None, 0, 1.0, 0.0) == -1
    assert lib.dsm_field_signed_enable(ctx.h) == -7                  # before dsm_field_enable
    assert lib.dsm_field_signed(ctx.h, None) == -7
    ctx.field_enable(0.1, 16, 16, 8)
    ctx.field_query_enable(16, 4, 16)
    assert query(ctx) == -7                                          # no field request yet
    ctx.field_enqueue((0, 0, 0), 5)                                  # a request without the signed grid
    assert lib.dsm_field_signed_enable(ctx.h) == -7                  # while a field is in flight
    ctx.field_wait()
    assert lib.dsm_field_signed(ctx.h, capi.ctypes.byref(P3)) == -7  # the waited request has no signed grid
    assert query(ctx) == -7                                          # nor has the latest request
    assert lib.dsm_field_signed_enable(ctx.h) == 0
    assert lib.dsm_field_signed_enable(ctx.h) == -7                  # once
    assert lib.dsm_field_signed(ctx.h, None) == -7                   # the last waited request predates it
    assert query(ctx) == -7
    ctx.field_enqueue((0, 0, 0), 5, host_copy=False)
    assert lib.dsm_field_signed(ctx.h, None) == -7                   # not waited yet
    assert query(ctx) == 0                                           # the latest request has it, in flight or not
    assert query(ctx) == -7                                          # one query in flight
    assert lib.dsm_field_query_wait(ctx.h, None, None) == 0
    assert lib.dsm_field_query_enqueue_signed(ctx.h, pts.ctypes.data, -1, None, None, 0, 1.0, 0.0) == -1
    assert lib.dsm_field_query_enqueue_signed(ctx.h, pts.ctypes.data, 17, None, None, 0, 1.0, 0.0) == -1
    assert lib.dsm_field_query_enqueue_signed(ctx.h, None, 1, None, None, 0, 1.0, 0.0) == -1
    assert lib.dsm_field_query_enqueue_signed(ctx.h, pts.ctypes.data, 1, None, None, 0, 0.0, 0.0) == -1
    assert lib.dsm_field_query_enqueue_signed(ctx.h, pts.ctypes.data, 1, None, None, 0, 1.0, -1.0) == -1
    ctx.field_wait()
    P3 = capi.ctypes.c_void_p(1)
    assert lib.dsm_field_signed(ctx.h, capi.ctypes.byref(P3)) == 0 and P3.value is None   # resident: NULL
    ctx.field_enqueue((0, 0, 0), 5)
    assert lib.dsm_field_signed(ctx.h, None) == -7                   # valid until the next field enqueue
    ctx.field_wait()
    assert lib.dsm_field_signed(ctx.h, capi.ctypes.byref(P3)) == 0 and P3.value
    ctx.close()


# ---- the node ----


def test_node_signed_field_equals_the_oracle_and_changes_nothing(tmp_path):
    """The node drive (keyframes, loop closures): every fused frame's signed grid and signed queries equal the oracle
    over the node's own clouds (a plain field of surfaces: its sites lie one voxel deep, so the test asks for no
    negative value); distances, clouds, PLY and PCD files equal a twin without the signed grid."""
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    node = [2, 0, 1 << 20, 1 << 21]
    r = run_driver("field_signed_main", str(tmp_path), cam, sc, node + [1, *NODE_FIELD], tag="a", after=[pa])
    q = run_driver("field_signed_main", str(tmp_path), cam, sc, node + [0, *NODE_FIELD], tag="b", after=[pb])
    for t in range(n):
        rc = r.i()
        c = r.take(np.float64, 3).copy()
        origin, n_occ = r.take(np.int32, 3).copy(), r.i()
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        rsg, sdist = r.i(), r.lst(np.float32).reshape(nz, ny, nx)
        rs, pts, samples = r.i(), r.lst(np.float64).reshape(-1, 3), r.lst(fq.SAMPLE_DTYPE)
        rt = r.i()
        step, radius = r.take(np.float32, 2).copy()
        wp, ofs, clear = r.lst(np.float64).reshape(-1, 3), r.lst(np.int32), r.lst(fq.CLEARANCE_DTYPE)
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        qc = q.i()
        q.take(np.float64, 3), q.take(np.int32, 3), q.i()
        qdist = q.lst(np.float32).reshape(nz, ny, nx)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == rsg == rs == rt == rr == qc == rq == 0, f"message {t}"
        wd, ws, o, wn = fs.field(xyz(act, inact), voxel, (nx, ny, nz), c)
        assert origin.tolist() == o.tolist() and n_occ == wn, f"message {t}: field"
        assert dist.tobytes() == wd.tobytes() == qdist.tobytes(), f"message {t}: dist"
        assert sdist.tobytes() == ws.tobytes(), f"message {t}: {differ(sdist, ws)} signed voxels differ"
        assert samples.tobytes() == fs.sample(ws, o, voxel, pts).tobytes(), f"message {t}: samples"
        assert clear.tobytes() == fs.clearance(ws, o, voxel, wp, ofs, step, radius).tobytes(), f"message {t}: clearance"
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.lst(POINT_DTYPE).tobytes() == q.lst(POINT_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
