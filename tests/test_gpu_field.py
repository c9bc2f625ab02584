"""dsm_field_enable / _enqueue / _wait: the map as a distance field, built in stream order.

Every field equals oracle/pyoracle_field applied to the synchronous readers (dsm_pool_export_cloud(m) +
dsm_inactive_export_cloud) at the same position in the stream, bit for bit, with the same origin and occupied count; the
field changes nothing in the map; the rejected-frame and error contracts; and dsm::SurfelMapNode::distance_field
(tests/cpp/field_main.cpp)."""
import filecmp

import numpy as np
import pytest

import pyoracle_field
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import (
    COMBOS, SHAPES, STORE, T, assert_field, camera, centres, field_points, map_state, new_ctx, simple_lists, warp, windowed,
    xyz)
from util import CAM

pytestmark = pytest.mark.gpu


def field_equals_oracle(ctx, voxel, shape, center, m, what):
    ctx.field_enqueue(center, m)
    got = ctx.field_wait()
    want = pyoracle_field.field(field_points(ctx, m), voxel, shape, center)
    assert_field(got, want, what)
    return got


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_field_equals_the_oracle_on_the_readers(chunk, shape):
    """The windowed drive of tests/test_gpu_publish.py with loop-closure warps between calls; after every call, one field
    per centre, the filter and the voxel edge cycling through {1, 5} x {0.125, 0.1, 0.3}."""
    lists = simple_lists()
    seen = {"empty": 0, "occupied": 0, "stored": 0}
    ctxs = {}   # one context per voxel edge: the grid is fixed at enable time
    for _, voxel in COMBOS:
        if voxel not in ctxs:
            ctxs[voxel] = new_ctx(store=STORE)
            ctxs[voxel].field_enable(voxel, *shape)
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c in ctxs.values():
            windowed(c, t0, t1, lists, want_counts=False)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:   # a loop closure between two calls
            for c in ctxs.values():
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
        for j in range(4):
            m, voxel = COMBOS[(call * 4 + j) % len(COMBOS)]
            ctx = ctxs[voxel]
            name, c = centres(ctx, t1 - 1, voxel, shape, m)[j]
            if c is None:
                continue
            got = field_equals_oracle(ctx, voxel, shape, c, m, f"frames {t0}-{t1 - 1}, m={m}, voxel={voxel}, {name}")
            if name == "off the map":
                assert got[2] == 0 and np.isposinf(got[0]).all()
            if name == "on an obstacle":
                assert got[2] > 0 and got[0].min() == 0.0
            seen["empty" if got[2] == 0 else "occupied"] += 1
            seen["stored"] += ctx.inactive_size()[0] > 0
    assert seen["occupied"] and seen["empty"] and seen["stored"], seen
    for c in ctxs.values():
        c.close()


def test_field_of_a_size_a_user_runs():
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    shape, voxel = (320, 320, 40), 0.1
    ctx.field_enable(voxel, *shape)
    windowed(ctx, 0, T, lists, want_counts=False)
    got = field_equals_oracle(ctx, voxel, shape, camera(T - 1), 5, "320x320x40 at the end of the drive")
    assert got[2] > 0 and np.isfinite(got[0]).all()
    ctx.close()


def test_field_beside_a_publish_snapshot_and_an_asynchronous_checkpoint(tmp_path):
    lists = simple_lists()
    ctx = new_ctx(store=STORE)
    shape, voxel = (64, 64, 32), 0.125
    ctx.field_enable(voxel, *shape)
    ctx.publish_enable()
    ctx.checkpoint_enable()
    windowed(ctx, 0, 10, lists, want_counts=False)
    ctx.publish_enqueue(5)
    ctx.checkpoint_enqueue(str(tmp_path / "async.dsm"))
    ctx.field_enqueue(camera(9), 5)
    ctx.inactive_transform(1, warp(2))   # enqueued behind all three: none of them sees it
    ctx.pool_transform(warp(1))
    got = ctx.field_wait()
    active, inactive, _ = ctx.publish_wait()
    assert ctx.checkpoint_wait(True)
    ref = new_ctx(store=STORE)
    windowed(ref, 0, 10, lists, want_counts=False)
    assert_field(got, pyoracle_field.field(field_points(ref, 5), voxel, shape, camera(9)), "field")
    assert active.tobytes() == ref.pool_export_cloud(5).tobytes() and inactive.tobytes() == ref.inactive_export_cloud().tobytes()
    ref.map_save(str(tmp_path / "sync.dsm"))
    assert filecmp.cmp(str(tmp_path / "async.dsm"), str(tmp_path / "sync.dsm"), shallow=False)
    assert len(inactive) > 0
    ctx.close()
    ref.close()


@pytest.mark.parametrize("chunk", [1, 4])
def test_fields_change_nothing_in_the_map(chunk):
    lists = simple_lists()
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    a.field_enable(0.1, 64, 64, 32)
    for c in (a, b):
        c.publish_enable()
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for c in (a, b):
            windowed(c, t0, t1, lists, want_counts=False)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        a.field_enqueue(camera(t1 - 1), 5)
        if call % 2 == 1 and stored:
            for c in (a, b):
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
        for c in (a, b):
            c.publish_enqueue(5)
        pa, pb = a.publish_wait(), b.publish_wait()
        a.field_wait()
        what = f"after frames {t0}-{t1 - 1}"
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes(), f"{what}: published clouds"
        assert map_state(a) == map_state(b), f"{what}: pool, store or table"
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_wait_and_stays_for_the_next_read():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    a = new_ctx(store=STORE)
    windowed(a, 0, first, lists, want_counts=False)
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    windowed(b, 0, first + 2, lists, want_counts=False)
    b.field_enqueue(camera(first - 1), 1)
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6
    want = pyoracle_field.field(field_points(a, 1), voxel, shape, camera(first - 1))
    assert_field(e.value.field, want, "field after the rejected frame")
    assert want[2] > 0
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    assert b.pool_size() == a.pool_size()
    b.field_enqueue(camera(first - 1), 1)
    assert_field(b.field_wait(), want, "field after the error was cleared")
    a.close()
    b.close()


def test_error_contract(tmp_path):
    lib = capi.load_library()
    P = capi.DsmFieldParams

    def C(*v):
        return (capi.ctypes.c_double * 3)(*v)

    bare = capi.Context(CAM, max_batch=1, max_local_surfels=1 << 16)
    assert lib.dsm_field_enable(bare.h, capi.ctypes.byref(P(0.1, 8, 8, 8))) == -7   # no resident pool
    bare.close()
    ctx = new_ctx(store=STORE)
    assert lib.dsm_field_enqueue(ctx.h, C(0, 0, 0), 5) == -7                        # before enable
    assert lib.dsm_field_wait(ctx.h, None, None, None) == -7
    for bad in [P(0.0, 8, 8, 8), P(-0.1, 8, 8, 8), P(float("nan"), 8, 8, 8), P(float("inf"), 8, 8, 8),
                P(0.1, 0, 8, 8), P(0.1, 8, 1025, 8), P(0.1, 8, 8, -1)]:
        assert lib.dsm_field_enable(ctx.h, capi.ctypes.byref(bad)) == -1
    assert lib.dsm_field_enable(ctx.h, None) == -1
    assert lib.dsm_field_enable(None, capi.ctypes.byref(P(0.1, 8, 8, 8))) == -1
    ctx.field_enable(0.5, 16, 16, 8)
    assert lib.dsm_field_enable(ctx.h, capi.ctypes.byref(P(0.1, 8, 8, 8))) == -7     # once
    assert lib.dsm_field_wait(ctx.h, None, None, None) == -7                         # nothing enqueued
    assert lib.dsm_field_enqueue(ctx.h, C(0, 0, 0), 0) == -1                         # min_update_times < 1
    assert lib.dsm_field_enqueue(ctx.h, None, 5) == -1
    for c in [(float("nan"), 0, 0), (0, float("inf"), 0), (0, 0, -float("inf")), (0.5 * 2 ** 24, 0, 0), (0, -0.5 * 2 ** 24, 0), (1e300, 0, 0)]:
        assert lib.dsm_field_enqueue(ctx.h, C(*c), 5) == -1, c
    assert lib.dsm_field_enqueue(ctx.h, C(0.5 * (2 ** 24 - 16), 0, 0), 5) == 0        # just inside the bound
    assert lib.dsm_field_wait(ctx.h, None, None, None) == 0                          # every out-pointer may be NULL
    windowed(ctx, 0, 8, simple_lists(), want_counts=False)
    ctx.map_save(str(tmp_path / "m.dsm"))
    surfels, segs = ctx.inactive_download(-1), ctx.inactive_segments()
    ctx.field_enqueue(camera(7), 5)
    assert lib.dsm_field_enqueue(ctx.h, C(0, 0, 0), 5) == -7                         # one field in flight
    assert lib.dsm_inactive_reserve(ctx.h, 1000) == -7
    with pytest.raises(capi.DsmError) as e:
        ctx.inactive_load(surfels, segs)
    assert e.value.code == -7
    with pytest.raises(capi.DsmError) as e:
        ctx.map_load(str(tmp_path / "m.dsm"))
    assert e.value.code == -7
    with pytest.raises(capi.DsmError) as e:
        ctx.map_load_journal(str(tmp_path / "m.dsm"))
    assert e.value.code == -7
    got = ctx.field_wait()
    assert_field(got, pyoracle_field.field(field_points(ctx, 5), 0.5, (16, 16, 8), camera(7)), "field after the refused calls")
    assert lib.dsm_field_wait(ctx.h, None, None, None) == -7                         # retired
    ctx.inactive_load(surfels, segs)                                                 # nothing in flight: allowed again
    ctx.map_load(str(tmp_path / "m.dsm"))
    ctx.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)


@pytest.mark.parametrize("publish", [0, 1])
def test_node_field_equals_the_oracle_and_changes_nothing(tmp_path, publish):
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("field_main", str(tmp_path), cam, sc, [2, 0, 1 << 20, 1 << 21, publish, *FIELD], tag="a", after=[pa])
    q = run_driver("field_main", str(tmp_path), cam, sc, [2, 0, 1 << 20, 1 << 21, publish, 0.0, 1, 1, 1], tag="b", after=[pb])
    occupied = 0
    for t in range(n):
        rc = r.i()
        c = r.take(np.float64, 3).copy()
        origin, n_occ = r.take(np.int32, 3).copy(), r.i()
        dist = r.lst(np.float32).reshape(nz, ny, nx)
        pub = [(r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)) for _ in range(publish)]
        pub_q = [(q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)) for _ in range(publish)]
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == 0 and rr == 0 and rq == 0, f"message {t}"
        want = pyoracle_field.field(xyz(act, inact), voxel, (nx, ny, nz), c)
        assert_field((dist, origin, n_occ), want, f"message {t}")
        occupied += n_occ > 0
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
        for (ra, a1, b1), (rb, a2, b2) in zip(pub, pub_q):
            assert ra == rb == 0 and a1.tobytes() == a2.tobytes() == act.tobytes() and b1.tobytes() == b2.tobytes() == inact.tobytes()
    assert occupied > n // 2
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.lst(POINT_DTYPE).tobytes() == q.lst(POINT_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
