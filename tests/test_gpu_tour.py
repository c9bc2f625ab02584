"""dsm_tour_enable / _enqueue / _wait: the order of an exploration tour, by a multi-start local search over a travel-cost
matrix.

The device equals oracle/pyoracle_tour.tour bit for bit in the header, every start record and the order: on random
asymmetric matrices at n = 1, 2, 3, 4, 17, 64, 200 and 1024 (the last at the passes the work bound allows), with and
without UINT32_MAX entries, open and closed; on symmetric and stretched metric matrices; with n_starts from 1 to
max_starts; on the matrices of matrix jobs over the windowed drive's known fields.  One job in flight, a wait that
waits for its own job only, a drive with tour jobs beside publish snapshots, checkpoints and matrix jobs against a twin
without them, and every error code.  The node is checked through tests/cpp/tour_main.cpp."""
import filecmp

import numpy as np
import pytest

import pyoracle_reach_matrix as RM
import pyoracle_tour as TM
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import STORE, T, camera, map_state, new_ctx, simple_lists, warp, windowed
from test_gpu_field_known import MAX_RANGE, Views
from test_tour_model import metric_matrix, random_matrix

pytestmark = pytest.mark.gpu

SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)


def context(max_sites, max_starts):
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.tour_enable(max_sites, max_starts)
    return ctx


def same(got, want, what):
    gi, gs, go = got
    wi, ws, wo = want
    assert gi.tobytes() == np.array(wi).tobytes(), f"{what}: header {gi} want {wi}"
    assert gs.tobytes() == ws.tobytes(), f"{what}: starts\n{gs}\nwant\n{ws}"
    assert go.tobytes() == wo.tobytes(), f"{what}: order\n{go}\nwant\n{wo}"


def job(ctx, M, open_, n_starts, max_passes, seed, what=""):
    ctx.tour_enqueue(M, open_, n_starts, max_passes, seed)
    got = ctx.tour_wait()
    same(got, TM.tour(M, open_, n_starts, max_passes, seed), what)
    return got


@pytest.mark.parametrize("n", [1, 2, 3, 4, 17, 64, 200])
def test_random_matrices(n):
    ctx = context(200, 64)
    rng = np.random.default_rng(n)
    for open_ in (0, 1):
        for p_inf in (0.0, 0.05, 0.4):
            for sym in (False, True):
                M = random_matrix(n, rng, p_inf, sym, hi=int(rng.choice([4, 1000, 1 << 31])))
                k = int(rng.integers(1, 65 if n <= 64 else 9))
                job(ctx, M, open_, k, 4096 if n <= 64 else 1000, int(rng.integers(0, 1 << 63)), f"n={n} open={open_} p_inf={p_inf} sym={sym} starts={k}")
        job(ctx, metric_matrix(n, rng), open_, 16 if n <= 64 else 4, 4096 if n <= 64 else 1000, n, f"metric n={n} open={open_}")
    ctx.close()


def test_1024_sites_at_the_work_bound():
    """n = 1024 with 4 starts at 1024 passes (4 x 1024 x 1024^2 = 2^32), and 1 start at 4096; a pass cut of 3."""
    ctx = context(1024, 4)
    rng = np.random.default_rng(1024)
    M = random_matrix(1024, rng)
    job(ctx, M, 0, 4, 1024, 5, "1024 closed")
    job(ctx, metric_matrix(1024, rng), 1, 1, 4096, 6, "1024 metric open")
    Mi = random_matrix(1024, rng, 0.02)
    got = job(ctx, Mi, 1, 2, 3, 7, "1024 with UINT32_MAX, 3 passes")
    assert (got[1]["passes"] == 3).all() and (got[1]["converged"] == 0).all()
    ctx.close()


def test_every_start_count():
    """n_starts from 1 to max_starts on one matrix: each start's record does not depend on how many starts run."""
    ctx = context(40, 1024)
    rng = np.random.default_rng(3)
    M = random_matrix(40, rng, 0.02)
    full = job(ctx, M, 0, 1024, 64, 9, "1024 starts")
    for k in (1, 2, 31, 32, 33, 255, 256, 257, 1023):
        ctx.tour_enqueue(M, 0, k, 64, 9)
        info, starts, order = ctx.tour_wait()
        best = int(np.lexsort((np.arange(k), full[1]["cost"][:k]))[0])
        assert starts.tobytes() == full[1][:k].tobytes() and info["best_start"] == best, k
        assert info["best_cost"] == full[1]["cost"][best] and info["n_starts"] == k and order[0] == 0, k
    assert (full[1]["cost"][1:] < full[1]["cost"][0]).any()      # some start beats nearest neighbour
    ctx.close()


def test_matrices_of_the_drive():
    """The windowed drive with loop-closure warps: after every call a known field, its frontiers, a reach job from the
    camera to the clusters and a matrix job over the camera, the field's centre and the reached viewpoints; the tour
    over that matrix as it stands equals the model, open and closed."""
    lists = simple_lists()
    shape, v = (64, 64, 32), 0.1
    ctx = new_ctx(store=STORE)
    ctx.field_enable(v, *shape)
    views = Views(ctx, 6)
    ctx.frontier_enable(64, 1 << 16)
    ctx.reach_enable(31, 1 << 12, 2048)
    ctx.reach_matrix_enable(32, 8 * 8 * 4, 2048)
    ctx.tour_enable(32, 64)
    stored, seen = set(), 0
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        windowed(ctx, t0, t1, lists, want_counts=False)
        views.capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            ctx.pool_transform(warp(1))
            ctx.inactive_transform(max(stored), warp(2))
            views.warp(warp(1))
        slots, poses = views.request()
        cam = camera(t1 - 1)
        ctx.field_enqueue_known(cam, 5, slots, poses)
        _, origin, _ = ctx.field_wait()
        ctx.frontier_enqueue(1)
        ctx.frontier_wait()
        ctx.reach_enqueue(cam, 0.0, 1, None, True)
        _, targets, _, _ = ctx.reach_wait()
        nx, ny = shape[0], shape[1]
        vp = targets["viewpoint"][targets["status"] == 0][:30].astype(np.int64)
        pts = [tuple(cam), tuple((np.array(origin) + np.array(shape) // 2 + 0.5) * float(np.float32(v)))]
        pts += [tuple((np.array(origin) + [x % nx, x // nx % ny, x // (nx * ny)] + 0.5) * float(np.float32(v))) for x in vp.tolist()]
        ctx.reach_matrix_enqueue(pts, 0.0, 1)
        _, _, M = ctx.reach_matrix_wait()
        for open_ in (0, 1):
            got = job(ctx, M, open_, 64, 256, call, f"call {call} open={open_}")
            seen += int(got[0]["n_included"]) > 3
    assert seen > 0
    ctx.close()


def test_one_job_in_flight_and_its_own_wait():
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.2, 40, 30, 20)
    ctx.views_enable(1, 1.0)
    ctx.reach_matrix_enable(8, 5 * 4 * 3, 256)
    ctx.tour_enable(64, 8)
    rng = np.random.default_rng(2)
    M = random_matrix(64, rng)
    st = rng.choice(3, size=(20, 30, 40), p=(0.1, 0.1, 0.8)).astype(np.uint8)
    ctx.debug_field_load_state(st, (0, 0, 0))
    dist = ctx.field_wait()[0]
    pts = rng.uniform(0, 4, size=(8, 3))
    ctx.reach_matrix_enqueue(pts, 0.0, 1)
    ctx.tour_enqueue(M, 0, 8, 64, 1)
    with pytest.raises(capi.DsmError) as e:
        ctx.tour_enqueue(M, 0, 8, 64, 1)
    assert e.value.code == -7
    same(ctx.tour_wait(), TM.tour(M, 0, 8, 64, 1), "tour before the matrix wait")
    RMw = RM.matrix(st, dist, (0, 0, 0), 0.2, pts, 0.0, 1, 5 * 4 * 3, 256)
    got = ctx.reach_matrix_wait()                        # the matrix job is still waiting for its own wait
    assert all(x.tobytes() == np.array(y).tobytes() for x, y in zip(got, RMw))
    with pytest.raises(capi.DsmError) as e:
        ctx.tour_wait()
    assert e.value.code == -7
    ctx.tour_enqueue(got[2], 1, 3, 16, 2)
    same(ctx.tour_wait(), TM.tour(got[2], 1, 3, 16, 2), "the matrix job's output")
    ctx.close()


def test_tour_jobs_change_nothing_else(tmp_path):
    """A drive with frontier, reach and matrix jobs beside a publish snapshot and an asynchronous checkpoint, with tour
    jobs enqueued among them, leaves the map, the clouds, the fields, the frontiers, the reach and matrix results and the
    checkpoint files byte-identical to a twin without tour jobs."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    va, vb = {}, {}
    for c, d in ((a, va), (b, vb)):
        c.field_enable(voxel, *shape)
        c.publish_enable()
        c.checkpoint_enable()
        d["v"] = Views(c, 4)
        c.frontier_enable(32, 4096)
        c.reach_enable(64, 1 << 14, 1024)
        c.reach_matrix_enable(8, 8 * 8 * 4, 1024)
    a.tour_enable(256, 16)
    rng = np.random.default_rng(4)
    stored = set()
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        for c, d in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            d["v"].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        outs = []
        pts = [camera(t) for t in range(t1)][-8:]
        M = random_matrix(256, rng, 0.01)
        for c, d in ((a, va), (b, vb)):
            slots, poses = d["v"].request()
            c.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
            c.frontier_enqueue(1)
            c.reach_matrix_enqueue(pts, 0.1, 2)
            if c is a:
                a.tour_enqueue(M, call % 2, 16, 64, call)
            c.reach_enqueue(camera(t1 - 1), 0.1, 2, [camera(0)], True, True)
            c.publish_enqueue(5)
            c.checkpoint_enqueue(str(tmp_path / f"{'ab'[c is b]}{call}.dsm"))
            if call % 2 == 1 and stored:
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
                d["v"].warp(warp(1))
            f = c.field_wait()
            st = c.field_state()
            fr = c.frontier_wait()
            rm = c.reach_matrix_wait()
            re = c.reach_wait()
            p = c.publish_wait()
            assert c.checkpoint_wait(True)
            outs.append((f, st, p, fr, re, rm))
        what = f"after frames {t0}-{t1 - 1}"
        same(a.tour_wait(), TM.tour(M, call % 2, 16, 64, call), what)
        (fa, sa, pa, fra, rea, rma), (fb, sb, pb, frb, reb, rmb) = outs
        assert fa[0].tobytes() == fb[0].tobytes() and sa[0].tobytes() == sb[0].tobytes(), f"{what}: field"
        for x, y, name in ((fra, frb, "frontiers"), (rea, reb, "reach"), (rma, rmb, "matrix")):
            assert all(np.asarray(u).tobytes() == np.asarray(w).tobytes() for u, w in zip(x, y)), f"{what}: {name}"
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes(), f"{what}: clouds"
        assert map_state(a) == map_state(b), f"{what}: map"
        assert filecmp.cmp(str(tmp_path / f"a{call}.dsm"), str(tmp_path / f"b{call}.dsm"), shallow=False), f"{what}: checkpoint"
    a.close()
    b.close()


def test_error_contract():
    lib = capi.load_library()
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    m4 = np.zeros((4, 4), np.uint32)
    assert lib.dsm_tour_enqueue(ctx.h, m4.ctypes.data, 4, 0, 1, 1, 0) == -7        # before dsm_tour_enable
    assert lib.dsm_tour_wait(ctx.h, None, None, None) == -7
    for ms, mk in [(0, 1), (1025, 1), (-1, 1), (1, 0), (1, 1025), (1, -1)]:
        assert lib.dsm_tour_enable(ctx.h, ms, mk) == -1, (ms, mk)
    assert lib.dsm_tour_enable(None, 1, 1) == -1
    assert lib.dsm_tour_enable(ctx.h, 4, 3) == 0                                   # no field, no map needed
    assert lib.dsm_tour_enable(ctx.h, 4, 3) == -7                                  # once
    assert lib.dsm_tour_wait(ctx.h, None, None, None) == -7                        # nothing enqueued
    for mat, n, o, k, p in [(None, 4, 0, 1, 1), (m4, 0, 0, 1, 1), (m4, 5, 0, 1, 1), (m4, -1, 0, 1, 1), (m4, 4, 2, 1, 1),
                            (m4, 4, -1, 1, 1), (m4, 4, 0, 0, 1), (m4, 4, 0, 4, 1), (m4, 4, 0, 1, -1), (m4, 4, 0, 1, 65537)]:
        assert lib.dsm_tour_enqueue(ctx.h, None if mat is None else mat.ctypes.data, n, o, k, p, 0) == -1, (n, o, k, p)
    assert lib.dsm_tour_enqueue(None, m4.ctypes.data, 4, 0, 1, 1, 0) == -1
    assert lib.dsm_tour_enqueue(ctx.h, m4.ctypes.data, 4, 1, 3, 65536, 0) == 0     # 3 x 2^16 x 16 < 2^32
    assert lib.dsm_tour_enqueue(ctx.h, m4.ctypes.data, 4, 1, 3, 0, 0) == -7        # one job in flight
    info = np.zeros(1, capi.TOUR_INFO_DTYPE)
    assert lib.dsm_tour_wait(ctx.h, info.ctypes.data, None, None) == 0
    assert info[0]["n_sites"] == 4 and info[0]["best_cost"] == 0 and (info[0]["reserved"] == 0).all()
    assert lib.dsm_tour_wait(ctx.h, None, None, None) == -7
    ctx.close()
    # the work bound: n_starts x max_passes x n^2 above 2^32
    w = context(1024, 1024)
    big = np.zeros((1024, 1024), np.uint32)
    assert lib.dsm_tour_enqueue(w.h, big.ctypes.data, 1024, 0, 4, 1025, 0) == -1   # 4 x 1025 x 2^20 > 2^32
    assert lib.dsm_tour_enqueue(w.h, big.ctypes.data, 1024, 0, 1025, 4, 0) == -1   # past max_starts
    assert lib.dsm_tour_enqueue(w.h, big.ctypes.data, 1024, 0, 4, 1024, 0) == 0    # 2^32 exactly
    w.tour_wait()
    w.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)
MAX_VIEWS = 5


def test_node_tour_equals_the_model(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers(), reach(with_frontiers) from the
    field's centre, reach_matrix over that point and the reached viewpoints, and tour() over that matrix; every dumped
    tour equals the model on the dumped matrix."""
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    node = [2, 0, 1 << 20, 1 << 21, *FIELD, MAX_VIEWS, MAX_RANGE]
    r = run_driver("tour_main", str(tmp_path), cam, sc, node + [32, 12 * 12 * 4, 2048, 32, 512])
    found = 0
    for t in range(n):
        rc, open_ = r.i(), r.i()
        seed = int(r.take(np.uint64, 1)[0])
        M = r.lst(np.uint32)
        info = r.take(np.uint8, TM.INFO_DTYPE.itemsize).view(TM.INFO_DTYPE)[0].copy()
        starts = r.lst(TM.START_DTYPE)
        order = r.lst(np.int32)
        assert rc == 0, f"message {t}: {rc}"
        k = int(round(np.sqrt(len(M))))
        M = M.reshape(k, k)
        same((info, starts, order), TM.tour(M, open_, 32, 512, seed), f"message {t}")
        found += int(info["n_included"]) > 2
    assert found > 0
    assert r.o == len(r.raw)
