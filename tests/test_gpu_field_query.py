"""dsm_field_enqueue_resident and dsm_field_query_*: planner queries against the latest distance field, on the device.

Every query equals oracle/pyoracle_field_query applied to the field it read, bit for bit: on every field of the windowed
drive, at random points and at points exactly on voxel centres, faces and the grid's bounds; a resident field answers as
its host copy does; the query keeps the grid of its own request when the next field is enqueued behind it; queries
beside a snapshot and an asynchronous checkpoint; queries change nothing in the map, the clouds or the fields; the
rejected-frame and error contracts; planner sizes; and dsm::SurfelMapNode with a resident field
(tests/cpp/field_query_main.cpp)."""

import numpy as np
import pytest

import pyoracle_field
import pyoracle_field_query as fq
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import (
    COMBOS, SHAPES, STORE, T, assert_field, camera, centres, field_points, map_state, new_ctx, simple_lists, warp, windowed,
    xyz)

pytestmark = pytest.mark.gpu

CAPS = (4096, 64, 512)   # points, trajectories, waypoints


def query_points(rng, origin, voxel, shape, n=1500):
    """Random points in and around the box, plus every kind of exact point: voxel centres, voxel faces, the box's
    first and last centres and the doubles just beyond them, non-finite coordinates."""
    v = float(np.float32(voxel))
    o, n3 = np.asarray(origin, np.float64), np.array(shape, np.float64)
    rnd = (o - 1 + rng.random((n, 3)) * (n3 + 2)) * v
    cells = rng.integers(0, np.array(shape), (200, 3))
    centre = (cells + o + 0.5) * v
    face = (cells + o) * v
    lo, hi = (o + 0.5) * v, (o + n3 - 0.5) * v
    bounds = np.stack([lo, hi, np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf), np.where(np.arange(3) == 0, hi, lo)])
    bad = np.array([[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0]]) + lo
    return np.concatenate([rnd, centre, face, bounds, bad])


def query_trajectories(rng, origin, voxel, shape, n=48):
    """n trajectories of 1-12 waypoints over the box (some beyond it), one-waypoint ones and zero-length segments, and
    two through exact voxel centres (the only inside points of a grid with an axis of one voxel)."""
    v = float(np.float32(voxel))
    o, n3 = np.asarray(origin, np.float64), np.array(shape, np.float64)
    wps, ofs = [], [0]
    for j in range(n):
        k = 1 if j % 7 == 0 else int(rng.integers(2, 13))
        w = (o - 2 + rng.random((k, 3)) * (n3 + 4)) * v
        if k > 2 and j % 3 == 0:
            w[2] = w[1]
        wps.append(w)
        ofs.append(ofs[-1] + k)
    for k in (1, 2):
        wps.append((rng.integers(0, np.array(shape), (k, 3)) + o + 0.5) * v)
        ofs.append(ofs[-1] + k)
    return np.concatenate(wps), np.array(ofs, np.int32)


def expected(dist, origin, voxel, pts, wp, ofs, step, radius):
    return fq.sample(dist, origin, voxel, pts), fq.clearance(dist, origin, voxel, wp, ofs, step, radius)


def assert_query(got, want, what):
    s, c = got
    ws, wc = want
    assert s.tobytes() == ws.tobytes(), f"{what}: {(s.view(np.uint32) != ws.view(np.uint32)).any(1).sum() if s.size else 0} samples differ"
    assert c.tobytes() == wc.tobytes(), f"{what}: clearance {c[c != wc][:4]} want {wc[c != wc][:4]}"


def query(ctx, pts, wp, ofs, step, radius):
    ctx.field_query_enqueue(pts, wp, ofs, step, radius)
    return ctx.field_query_wait()


def query_equals_oracle(ctx, rng, field, voxel, shape, what):
    dist, origin, _ = field
    pts = query_points(rng, origin, voxel, shape)
    wp, ofs = query_trajectories(rng, origin, voxel, shape)
    step, radius = voxel / 2, 2.5 * voxel
    got = query(ctx, pts, wp, ofs, step, radius)
    assert_query(got, expected(dist, origin, voxel, pts, wp, ofs, step, radius), what)
    return got


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_queries_equal_the_oracle_on_every_field(chunk, shape):
    """The windowed drive of tests/test_gpu_field.py, loop-closure warps between calls; after every call one field per
    centre (filter and voxel edge cycling), each queried at points and trajectories."""
    rng = np.random.default_rng(11)
    lists = simple_lists()
    seen = {"inside": 0, "outside": 0, "hit": 0, "empty": 0}
    ctxs = {}
    for _, voxel in COMBOS:
        if voxel not in ctxs:
            ctxs[voxel] = new_ctx(store=STORE)
            ctxs[voxel].field_enable(voxel, *shape)
            ctxs[voxel].field_query_enable(*CAPS)
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c in ctxs.values():
            windowed(c, t0, t1, lists, want_counts=False)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            for c in ctxs.values():
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
        for j in range(4):
            m, voxel = COMBOS[(call * 4 + j) % len(COMBOS)]
            ctx = ctxs[voxel]
            name, c = centres(ctx, t1 - 1, voxel, shape, m)[j]
            if c is None:
                continue
            ctx.field_enqueue(c, m)
            field = ctx.field_wait()
            s, cl = query_equals_oracle(ctx, rng, field, voxel, shape, f"frames {t0}-{t1 - 1}, m={m}, voxel={voxel}, {name}")
            seen["inside"] += int((~np.isnan(s["dist"])).sum())
            seen["outside"] += int(np.isnan(s["dist"]).sum())
            seen["hit"] += int((cl["first_hit"] >= 0).sum())
            seen["empty"] += field[2] == 0
    assert all(seen.values()), seen
    for c in ctxs.values():
        c.close()


def test_resident_field_answers_as_its_host_copy():
    rng = np.random.default_rng(12)
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_query_enable(*CAPS)
    windowed(ctx, 0, 12, lists, want_counts=False)
    ctx.field_enqueue(camera(11), 5)
    host = ctx.field_wait()
    pts = query_points(rng, host[1], voxel, shape)
    wp, ofs = query_trajectories(rng, host[1], voxel, shape)
    a = query(ctx, pts, wp, ofs, voxel / 2, 0.3)
    ctx.field_enqueue(camera(11), 5, host_copy=False)
    res = ctx.field_wait()
    assert res[0] is None and res[1].tolist() == host[1].tolist() and res[2] == host[2] > 0
    b = query(ctx, pts, wp, ofs, voxel / 2, 0.3)
    assert_query(b, a, "resident against host copy")
    assert_query(b, expected(host[0], host[1], voxel, pts, wp, ofs, voxel / 2, 0.3), "resident against the oracle")
    ctx.close()


def test_a_query_keeps_the_grid_of_its_own_request():
    """A query in flight when the next field is enqueued reads the old grid; a query enqueued behind a field that has
    not been waited for reads that field."""
    rng = np.random.default_rng(13)
    lists = simple_lists()
    shape, voxel = (48, 40, 24), 0.125
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_query_enable(*CAPS)
    windowed(ctx, 0, 14, lists, want_counts=False)
    ctx.field_enqueue(camera(13), 5, host_copy=False)
    ctx.field_wait()
    want_a = pyoracle_field.field(field_points(ctx, 5), voxel, shape, camera(13))
    other = camera(13) + np.array([1.3, -0.7, 0.4])
    want_b = pyoracle_field.field(field_points(ctx, 1), voxel, shape, other)
    pts = np.concatenate([query_points(rng, want_a[1], voxel, shape), query_points(rng, want_b[1], voxel, shape)])
    wp, ofs = query_trajectories(rng, want_a[1], voxel, shape)
    ctx.field_query_enqueue(pts, wp, ofs, voxel / 2, 0.25)
    ctx.field_enqueue(other, 1, host_copy=False)           # behind the query in the stream
    got_a = ctx.field_query_wait()
    ctx.field_query_enqueue(pts, wp, ofs, voxel / 2, 0.25)  # the new field is not waited for yet
    got_b = ctx.field_query_wait()
    res = ctx.field_wait()
    assert res[0] is None and res[1].tolist() == want_b[1].tolist() and res[2] == want_b[2]
    assert_query(got_a, expected(want_a[0], want_a[1], voxel, pts, wp, ofs, voxel / 2, 0.25), "query before the next field")
    assert_query(got_b, expected(want_b[0], want_b[1], voxel, pts, wp, ofs, voxel / 2, 0.25), "query behind the next field")
    assert got_a[0].tobytes() != got_b[0].tobytes()
    ctx.close()


def test_queries_beside_a_publish_snapshot_and_an_asynchronous_checkpoint(tmp_path):
    import filecmp
    rng = np.random.default_rng(14)
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.125
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_query_enable(*CAPS)
    ctx.publish_enable()
    ctx.checkpoint_enable()
    windowed(ctx, 0, 10, lists, want_counts=False)
    ref = new_ctx(store=STORE)
    windowed(ref, 0, 10, lists, want_counts=False)
    want = pyoracle_field.field(field_points(ref, 5), voxel, shape, camera(9))
    pts = query_points(rng, want[1], voxel, shape)
    wp, ofs = query_trajectories(rng, want[1], voxel, shape)
    ctx.publish_enqueue(5)
    ctx.checkpoint_enqueue(str(tmp_path / "async.dsm"))
    ctx.field_enqueue(camera(9), 5, host_copy=False)
    ctx.field_query_enqueue(pts, wp, ofs, voxel / 2, 0.3)
    ctx.inactive_transform(1, warp(2))   # enqueued behind all four: none of them sees it
    ctx.pool_transform(warp(1))
    got = ctx.field_query_wait()
    field = ctx.field_wait()
    active, inactive, _ = ctx.publish_wait()
    assert ctx.checkpoint_wait(True)
    assert field[1].tolist() == want[1].tolist() and field[2] == want[2]
    assert_query(got, expected(want[0], want[1], voxel, pts, wp, ofs, voxel / 2, 0.3), "query")
    assert active.tobytes() == ref.pool_export_cloud(5).tobytes() and inactive.tobytes() == ref.inactive_export_cloud().tobytes()
    ref.map_save(str(tmp_path / "sync.dsm"))
    assert filecmp.cmp(str(tmp_path / "async.dsm"), str(tmp_path / "sync.dsm"), shallow=False)
    ctx.close()
    ref.close()


@pytest.mark.parametrize("chunk", [1, 4])
def test_queries_change_nothing_in_the_map_the_clouds_or_the_fields(chunk):
    rng = np.random.default_rng(15)
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.publish_enable()
    a.field_query_enable(*CAPS)
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c in (a, b):
            windowed(c, t0, t1, lists, want_counts=False)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        for c in (a, b):
            c.field_enqueue(camera(t1 - 1), 5)
        o = pyoracle_field.origin(camera(t1 - 1), voxel, shape)
        a.field_query_enqueue(query_points(rng, o, voxel, shape, 300), *query_trajectories(rng, o, voxel, shape, 16), voxel / 2, 0.3)
        if call % 2 == 1 and stored:
            for c in (a, b):
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
        for c in (a, b):
            c.publish_enqueue(5)
        a.field_query_wait()
        pa, pb = a.publish_wait(), b.publish_wait()
        fa, fb = a.field_wait(), b.field_wait()
        what = f"after frames {t0}-{t1 - 1}"
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes(), f"{what}: published clouds"
        assert_field(fa, fb, f"{what}: field")
        assert map_state(a) == map_state(b), f"{what}: pool, store or table"
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_the_query_wait():
    rng = np.random.default_rng(16)
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    a = new_ctx(store=STORE)
    windowed(a, 0, first, lists, want_counts=False)
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    b.field_query_enable(*CAPS)
    windowed(b, 0, first + 2, lists, want_counts=False)
    b.field_enqueue(camera(first - 1), 1, host_copy=False)
    want = pyoracle_field.field(field_points(a, 1), voxel, shape, camera(first - 1))
    pts = query_points(rng, want[1], voxel, shape)
    wp, ofs = query_trajectories(rng, want[1], voxel, shape)
    b.field_query_enqueue(pts, wp, ofs, voxel / 2, 0.3)
    with pytest.raises(capi.DsmError) as e:
        b.field_query_wait()
    assert e.value.code == -6
    assert_query(e.value.query, expected(want[0], want[1], voxel, pts, wp, ofs, voxel / 2, 0.3), "query after the rejected frame")
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6 and e.value.field[0] is None
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # neither wait cleared it
    assert b.pool_size() == a.pool_size()
    b.field_enqueue(camera(first - 1), 1, host_copy=False)
    b.field_wait()
    assert_query(query(b, pts, wp, ofs, voxel / 2, 0.3), expected(want[0], want[1], voxel, pts, wp, ofs, voxel / 2, 0.3),
                 "query after the error was cleared")
    a.close()
    b.close()


def test_error_contract():
    lib = capi.load_library()
    D, I = capi.ctypes.c_double, capi.ctypes.c_int32

    def arr(t, v):
        v = list(v)
        return (t * max(len(v), 1))(*v)

    def enq(ctx, pts, wp, ofs, step=0.1, radius=0.2):
        p = arr(D, np.ravel(pts))
        w = arr(D, np.ravel(wp))
        o = arr(I, ofs)
        return lib.dsm_field_query_enqueue(ctx.h, p if len(pts) else None, len(pts), w if len(wp) else None,
                                           o if len(ofs) else None, max(len(ofs) - 1, 0), step, radius)

    ctx = new_ctx(store=STORE)
    assert lib.dsm_field_query_enable(ctx.h, 8, 2, 8) == -7                       # before dsm_field_enable
    assert lib.dsm_field_query_enable(None, 8, 2, 8) == -1
    ctx.field_enable(0.25, 16, 16, 8)
    for bad in [(-1, 2, 8), (8, -1, 8), (8, 2, -1), (1 << 27, 2, 8)]:
        assert lib.dsm_field_query_enable(ctx.h, *bad) == -1, bad
    assert lib.dsm_field_query_wait(ctx.h, None, None) == -7                       # not enabled
    assert enq(ctx, [[0, 0, 0]], [], []) == -7
    ctx.field_query_enable(8, 2, 8)
    assert lib.dsm_field_query_enable(ctx.h, 8, 2, 8) == -7                       # once
    assert enq(ctx, [[0, 0, 0]], [], []) == -7                                     # no field requested yet
    assert lib.dsm_field_query_wait(ctx.h, None, None) == -7                       # nothing enqueued
    windowed(ctx, 0, 8, simple_lists(), want_counts=False)
    ctx.field_enqueue(camera(7), 5, host_copy=False)
    wp = np.array([[0.0, 0, 0], [1, 0, 0], [1, 1, 0], [2, 2, 2]])
    ok = (np.zeros((8, 3)), wp, [0, 2, 4])
    assert enq(ctx, *ok) == 0                                                      # behind the unwaited field
    assert enq(ctx, *ok) == -7                                                     # one query in flight
    assert lib.dsm_field_query_wait(ctx.h, None, None) == 0                        # out-pointers may be NULL
    assert lib.dsm_field_query_wait(ctx.h, None, None) == -7                       # retired
    field = ctx.field_wait()
    refused = {
        "too many points": (np.zeros((9, 3)), wp, [0, 2, 4]),
        "too many trajectories": ([], np.concatenate([wp, wp[:2]]), [0, 2, 3, 4]),
        "too many waypoints": ([], np.zeros((9, 3)), [0, 9]),
        "offsets not from 0": ([], wp, [1, 2, 4]),
        "offsets not rising": ([], wp, [0, 2, 2]),
        "NaN waypoint": ([], np.where(np.arange(12).reshape(4, 3) == 4, np.nan, wp), [0, 2, 4]),
        "infinite waypoint": ([], np.where(np.arange(12).reshape(4, 3) == 11, -np.inf, wp), [0, 2, 4]),
        "more than 2^26 samples": ([], np.array([[0.0, 0, 0], [2.0 ** 27 * 0.1, 0, 0]]), [0, 2]),
        "infinite length": ([], np.array([[-1e200, 0, 0], [1e200, 0, 0]]), [0, 2]),
    }
    for what, (p, w, o) in refused.items():
        assert enq(ctx, p, w, o) == -1, what
        if "too many" not in what:   # the oracle refuses the same requests (capacities are the library's)
            with pytest.raises(ValueError):
                fq.segment_counts(*fq.check_request(w, o, 0.1, 0.2), 0.1)
    for step, radius in [(0.0, 0.2), (-0.1, 0.2), (float("nan"), 0.2), (float("inf"), 0.2), (0.1, -1e-30), (0.1, float("nan")),
                         (0.1, float("inf"))]:
        assert enq(ctx, *ok, step=step, radius=radius) == -1, (step, radius)
    assert lib.dsm_field_query_enqueue(ctx.h, None, 1, None, None, 0, 0.1, 0.2) == -1          # NULL with a count
    assert lib.dsm_field_query_enqueue(ctx.h, None, -1, None, None, 0, 0.1, 0.2) == -1
    assert lib.dsm_field_query_enqueue(ctx.h, None, 0, None, None, 1, 0.1, 0.2) == -1
    assert lib.dsm_field_query_enqueue(None, None, 0, None, None, 0, 0.1, 0.2) == -1
    assert lib.dsm_field_query_wait(ctx.h, None, None) == -7                       # nothing refused was enqueued
    assert lib.dsm_field_query_enqueue(ctx.h, None, 0, None, None, 0, 0.1, 0.2) == 0            # an empty query
    s, c = capi.ctypes.c_void_p(), capi.ctypes.c_void_p()
    assert lib.dsm_field_query_wait(ctx.h, capi.ctypes.byref(s), capi.ctypes.byref(c)) == 0
    ctx.field_query_enqueue(*ok, 0.1, 0.2)
    got = ctx.field_query_wait()
    dist = pyoracle_field.field(field_points(ctx, 5), 0.25, (16, 16, 8), camera(7))
    assert field[1].tolist() == dist[1].tolist()
    assert_query(got, expected(dist[0], dist[1], 0.25, *ok, 0.1, 0.2), "query after the refused calls")
    ctx.close()


def test_queries_at_planner_sizes():
    """1 Mi points and 4 Ki trajectories of 32 waypoints at step v / 2 on a 320 x 320 x 40 grid at 0.2 m."""
    rng = np.random.default_rng(17)
    lists = simple_lists()
    shape, voxel = (320, 320, 40), 0.2
    ctx = new_ctx(store=STORE)
    ctx.field_enable(voxel, *shape)
    ctx.field_query_enable(1 << 20, 4096, 4096 * 32)
    windowed(ctx, 0, T, lists, want_counts=False)
    ctx.field_enqueue(camera(T - 1), 5, host_copy=False)
    _, origin, n_occ = ctx.field_wait()
    want = pyoracle_field.field(field_points(ctx, 5), voxel, shape, camera(T - 1))
    assert origin.tolist() == want[1].tolist() and n_occ == want[2] > 0
    o, n3 = origin.astype(np.float64), np.array(shape, np.float64)
    pts = (o - 1 + rng.random((1 << 20, 3)) * (n3 + 2)) * float(np.float32(voxel))
    wp = ((o + rng.random((4096, 1, 3)) * n3) + np.cumsum(rng.normal(0, 2, (4096, 32, 3)), 1)) * float(np.float32(voxel))
    ofs = np.arange(4097, dtype=np.int32) * 32
    got = query(ctx, pts, wp.reshape(-1, 3), ofs, voxel / 2, 0.5)
    assert_query(got, expected(want[0], want[1], voxel, pts, wp.reshape(-1, 3), ofs, voxel / 2, 0.5), "planner sizes")
    assert (~np.isnan(got[0]["dist"])).sum() > (1 << 19)
    ctx.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)


def test_node_queries_equal_the_oracle_and_change_nothing(tmp_path):
    import filecmp
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("field_query_main", str(tmp_path), cam, sc, [2, 0, 1 << 20, 1 << 21, 1, *FIELD], tag="a", after=[pa])
    q = run_driver("field_query_main", str(tmp_path), cam, sc, [2, 0, 1 << 20, 1 << 21, 0, 0.0, 1, 1, 1], tag="b", after=[pb])
    hits = 0
    for t in range(n):
        rc = r.i()
        c = r.take(np.float64, 3).copy()
        origin, n_occ = r.take(np.int32, 3).copy(), r.i()
        rs = r.i()
        pts = r.lst(np.float64).reshape(-1, 3)
        samples = r.lst(fq.SAMPLE_DTYPE)
        rt = r.i()
        step, radius = r.take(np.float32, 2).copy()
        wp, ofs = r.lst(np.float64).reshape(-1, 3), r.lst(np.int32)
        clear = r.lst(fq.CLEARANCE_DTYPE)
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == rs == rt == rr == rq == 0, f"message {t}"
        want = pyoracle_field.field(xyz(act, inact), voxel, (nx, ny, nz), c)
        assert origin.tolist() == want[1].tolist() and n_occ == want[2], f"message {t}: field"
        assert_query((samples, clear), expected(want[0], want[1], voxel, pts, wp, ofs, step, radius), f"message {t}")
        hits += int((clear["first_hit"] >= 0).sum())
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
    assert hits > 0
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.lst(POINT_DTYPE).tobytes() == q.lst(POINT_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
