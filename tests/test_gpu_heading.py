"""dsm_heading_enable / _enqueue / _wait: the camera's heading along trajectories, planned on the device.

Every header, record, sample and count equals oracle/pyoracle_heading bit for bit on the windowed drive's known fields
(chunks 1 and 4, with loop-closure warps between calls), on crafted state grids loaded at a range of 128 voxels under
both blocking rules, and on the optimised control points of trajectory jobs.  The counts equal a device gain job on the
poses [R_r | p_s]; a job in flight across the next field request reads the old grid; a drive with heading jobs leaves
the map, the fields, the state grids, the published clouds and the checkpoint files byte-identical to a twin's without
them.  The rejected-frame and error contracts, and dsm::SurfelMapNode (tests/cpp/heading_main.cpp)."""
import ctypes

import numpy as np
import pytest

import pyoracle_field_signed as fs
import pyoracle_gain as G
import pyoracle_heading as H
import pyoracle_trajectory as tj
from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import (FREE, K, NODE_FIELD, OCCUPIED, RELOAD, SMALL_CAM, UNKNOWN, assert_error_stays, gcam, known_drive,
                         node_args, rejected, rejected_known, same, small_ctx, twin_clouds, twin_drive, twin_node_tail)
from node_drive import node_script, run_driver
from planner_scenes import rotations, scene
from resident_map import camera, load_known

pytestmark = pytest.mark.gpu

NAMES = ("header", "records", "samples", "counts")
CAPS = (64, 1 << 14)


def device_equals_model(ctx, state, origin, voxel, cam, rot, Ks, pts, ofs, req, wu, wf, what):
    ctx.heading_enqueue(pts, ofs, cam, rot, Ks, req, wu, wf)
    got = ctx.heading_wait()
    want = H.job(state, origin, voxel, cam, rot, Ks, pts, ofs, req, wu, wf)
    same(got, want, what, NAMES)
    return got


def lines_through(rng, centres, voxel, n_points=(7, 9, 12), spread=6.0):
    """One trajectory per centre: a noisy line through it, `spread` voxels to either side."""
    v = float(np.float32(voxel))
    pts, ofs = [], [0]
    for j, c in enumerate(centres):
        N = n_points[j % len(n_points)]
        d = rng.standard_normal(3) * [1.0, 1.0, 0.2]
        d *= spread * v / np.linalg.norm(d)
        q = np.asarray(c, np.float64) + np.linspace(-1, 1, N)[:, None] * d + rng.standard_normal((N, 3)) * 0.3 * v
        pts.append(q)
        ofs.append(ofs[-1] + N)
    return np.concatenate(pts), np.array(ofs, np.int32)


def random_requests(rng, n, n_rot):
    rows = []
    for j in range(n):
        m = int(rng.integers(0, n_rot + 1)) if j % 3 == 2 else int(rng.integers(0, 3))
        rows.append((int(rng.integers(n_rot)), int(rng.integers(-1, n_rot)) if j % 2 else -1, m))
    return H.requests(rows)


@pytest.mark.parametrize("chunk", [1, 4])
def test_drive_known_fields_equal_the_model(chunk):
    """The windowed drive with warps between calls: after every call, trajectories through the camera and beside it,
    scored at 8 or 16 yaws and two pitches against the known field at the camera, under both blocking rules."""
    rng = np.random.default_rng(chunk)
    planned = 0
    for call, t0, t1, ctx, v, cam, slots, poses, (_, origin, _), state in known_drive((64, 64, 32), chunk, (0.125, 0.1),
                                                                                     lambda c: c.heading_enable(*CAPS)):
        n_yaw = (8, 16)[call % 2]
        rot = rotations(n_yaw, (0.0, -0.3))[:max(n_yaw, 12)]
        gc = gcam(K, (10 + 5 * (call % 3)) * np.float32(v), call % 2)
        pts, ofs = lines_through(rng, [cam, cam + [4 * v, -3 * v, 0.0], cam + [-30 * v, 0, 0]], v, (7, 9, 7))
        req = random_requests(rng, 3, len(rot))
        got = device_equals_model(ctx, state, origin, v, gc, rot, 1 + call % 3, pts, ofs, req, 1 + call, 7,
                                  f"frames {t0}-{t1 - 1}, voxel {v}")
        planned += int((got[1]["score"] > 0).sum())
    assert planned > 0


def crafted(shape, rng):
    nx, ny, nz = shape
    slab = np.full(shape[::-1], FREE, np.uint8)
    slab[:, 2 * ny // 3:, :] = UNKNOWN
    slab[:, :, nx // 2] = np.where(np.arange(ny)[None, :] % 5 == 0, OCCUPIED, FREE)
    return {"slab": slab, "scene": scene(rng, shape, n_blobs=10, p_occupied=0.03),
            "random": rng.choice([UNKNOWN, OCCUPIED, FREE], size=shape[::-1], p=[0.15, 0.05, 0.8]).astype(np.uint8)}


def loaded_ctx(shape, voxel):
    ctx = small_ctx(shape, voxel)
    ctx.heading_enable(*CAPS)
    ctx.gain_enable(1 << 14)
    return ctx


@pytest.mark.parametrize("unknown_blocks", [0, 1])
def test_loaded_grids_at_128_voxels_equal_the_model_and_gain_jobs(unknown_blocks):
    """Crafted grids loaded as the latest known field, the camera's range at the cap of 128 voxels; the counts also
    equal a device gain job on every pose [R_r | p_s]."""
    shape, voxel, origin = (40, 32, 12), 0.1, (-20, -16, -6)
    rng = np.random.default_rng(40 + unknown_blocks)
    ctx = loaded_ctx(shape, voxel)
    v = float(np.float32(voxel))
    for name, st in crafted(shape, rng).items():
        load_known(ctx, st, origin, voxel, name)
        for max_range, n_yaw in ((128 * np.float32(v), 16), (25 * np.float32(v), 8)):
            gc = gcam(K, max_range, unknown_blocks)
            rot = rotations(n_yaw)
            centres = [np.zeros(3), [0.8, -0.5, 0.1], [-1.5, 1.2, -0.2], [3.0, 0.0, 0.0]]   # the last leaves the grid
            pts, ofs = lines_through(rng, centres, voxel, spread=10.0)
            req = random_requests(rng, len(centres), n_yaw)
            what = f"{name} range {max_range / v:.0f} voxels"
            info, recs, samples, counts = device_equals_model(ctx, st, origin, voxel, gc, rot, 2, pts, ofs, req, 2, 5, what)
            assert recs["n_outside"].sum() > 0, what
            if max_range > 25 * np.float32(v):
                continue   # a gain job refuses more than 123 views at 128 voxels
            poses = np.array([np.concatenate([R.reshape(3, 3), p[:, None]], axis=1).reshape(12) for p in samples["p"] for R in rot])
            ctx.gain_enqueue(gc, poses)
            _, g = ctx.gain_wait()
            g = g.reshape(counts.shape)
            assert (g["n_unknown"] == counts["n_unknown"]).all() and (g["n_frontier"] == counts["n_frontier"]).all(), what
    ctx.close()


def test_trajectory_job_outputs_equal_the_model():
    """The optimised control points of a trajectory job on the same loaded field, passed on unchanged."""
    shape, voxel, origin = (48, 32, 16), 0.1, (-24, -16, -8)
    rng = np.random.default_rng(3)
    ctx = small_ctx(shape, voxel)
    ctx.field_signed_enable()
    ctx.trajectory_enable(16, 4096, 8)
    ctx.heading_enable(*CAPS)
    st = crafted(shape, rng)["scene"]
    load_known(ctx, st, origin, voxel, "scene")
    sdist = ctx.field_signed()
    pts, ofs = lines_through(rng, [np.zeros(3), [0.5, 0.5, 0.0], [-0.8, 0.3, 0.1], [1.0, -0.6, 0.0]], voxel, (9, 16, 33, 64), 12.0)
    p = tj.params(margin=0.3, max_iter=30, samples=4)
    ctx.trajectory_enqueue(pts, ofs, np.full(len(ofs) - 1, 0.5), p)
    _, rec, out = ctx.trajectory_wait()
    wq, _, _ = tj.job(pts, ofs, np.full(len(ofs) - 1, 0.5), p, sdist, origin, voxel)
    assert out.tobytes() == wq.tobytes()
    rot = rotations(16)
    for ub in (0, 1):
        got = device_equals_model(ctx, st, origin, voxel, gcam(K, 20 * 0.1, ub), rot, 4, out, ofs,
                                  H.requests([(0, -1, 1), (4, 8, 2), (15, 0, 1), (3, -1, 16)]), 3, 1, f"trajectory outputs, ub {ub}")
        assert (got[2]["p"].reshape(-1, 3) == H.sample_positions(out, ofs, 4)).all()
    ctx.close()


def test_a_job_in_flight_reads_the_old_grid():
    shape, voxel, origin = (32, 32, 12), 0.1, (-16, -16, -6)
    rng = np.random.default_rng(2)
    ctx = loaded_ctx(shape, voxel)
    grids = crafted(shape, rng)
    load_known(ctx, grids["scene"], origin, voxel, "scene")
    pts, ofs = lines_through(rng, [np.zeros(3), [0.4, 0.4, 0.0]], voxel)
    gc, rot, req = gcam(K, 2.0, 1), rotations(8), H.requests([(0, -1, 1), (2, 6, 2)])
    ctx.heading_enqueue(pts, ofs, gc, rot, 3, req, 1, 1)
    ctx.debug_field_load_state(grids["random"], (3, 4, 5))    # the next request, before the job's wait
    got = ctx.heading_wait()
    same(got, H.job(grids["scene"], origin, voxel, gc, rot, 3, pts, ofs, req, 1, 1), "in flight", NAMES)
    ctx.field_wait()
    ctx.close()


def test_heading_jobs_change_nothing_else(tmp_path):
    """A drive with heading jobs beside a publish snapshot and an asynchronous checkpoint leaves the map, both published
    clouds, the fields, the state grids and the checkpoint files byte-identical to a twin without them."""
    rng = np.random.default_rng(5)
    job = {}

    def enqueue(c, is_a, call, t1):
        if is_a:
            cam = camera(t1 - 1)
            job["pts"], job["ofs"] = lines_through(rng, [cam, cam + [0.5, 0.3, 0.0]], 0.1)
            job["gc"], job["rot"], job["req"] = gcam(K, 20 * 0.1, call % 2), rotations(8), H.requests([(0, -1, 1), (3, 7, 2)])
            c.heading_enqueue(job["pts"], job["ofs"], job["gc"], job["rot"], 2, job["req"], 1, 3)

    def check(a, outs, call, t1, what):
        same(a.heading_wait(), H.job(outs["state"][0], outs["field"][1], 0.1, job["gc"], job["rot"], 2, job["pts"], job["ofs"],
                                     job["req"], 1, 3), what, NAMES)

    twin_drive(tmp_path, lambda c: None, lambda a: a.heading_enable(*CAPS), enqueue, lambda c: {}, check)


def test_rejected_frame_comes_back_from_wait():
    job = {}

    def enqueue(b, first):
        cam = camera(first - 1)
        job["pts"], job["ofs"] = lines_through(np.random.default_rng(1), [cam], 0.1)
        job["gc"], job["rot"], job["req"] = gcam(K, 30 * 0.1, 0), rotations(8), H.requests([(0, -1, 2)])
        b.heading_enqueue(job["pts"], job["ofs"], job["gc"], job["rot"], 3, job["req"], 1, 1)

    r = rejected_known(lambda b: b.heading_enable(4, 1024), enqueue)
    e = rejected(r.ctx.heading_wait)
    same(e.heading, H.job(r.state, r.field[1], r.voxel, job["gc"], job["rot"], 3, job["pts"], job["ofs"], job["req"], 1, 1),
         "rejected", NAMES)
    assert e.heading[3]["n_unknown"].sum() + e.heading[3]["n_frontier"].sum() > 0
    assert_error_stays(r.ctx)
    r.ctx.close()


def test_error_contract():
    lib = capi.load_library()
    cam = capi.DsmGainCamera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    rot = np.ascontiguousarray(rotations(4))
    pts = np.zeros((8, 3))
    pts[:, 0] = np.linspace(0.1, 0.7, 8)
    ofs = np.array([0, 8], np.int32)
    req = H.requests([(0, -1, 1)])

    def enq(ctx, c=cam, q=pts, o=ofs, n=1, r=rot, n_rot=4, k=2, rq=req, wu=1, wf=1):
        return lib.dsm_heading_enqueue(ctx.h, q.ctypes.data, o.ctypes.data, n, ctypes.byref(c), r.ctypes.data, n_rot, k, rq.ctypes.data,
                                       wu, wf)

    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    assert lib.dsm_heading_enable(None, 1, 1) == -1
    assert lib.dsm_heading_enqueue(None, None, None, 0, None, None, 0, 0, None, 0, 0) == -1
    assert lib.dsm_heading_wait(None, None, None, None, None) == -1
    assert lib.dsm_heading_enable(ctx.h, 4, 64) == -7                 # before dsm_field_enable
    ctx.field_enable(0.1, 16, 16, 8)
    assert lib.dsm_heading_enable(ctx.h, 4, 64) == -7                 # before dsm_views_enable
    ctx.views_enable(1, 1.0)
    assert enq(ctx) == -7                                             # before dsm_heading_enable
    assert lib.dsm_heading_wait(ctx.h, None, None, None, None) == -7
    for args in ((0, 64), (4, 0), ((1 << 22) + 1, 64), (4, (1 << 22) + 1)):
        assert lib.dsm_heading_enable(ctx.h, *args) == -1
    assert lib.dsm_heading_enable(ctx.h, 4, 64) == 0
    assert lib.dsm_heading_enable(ctx.h, 4, 64) == -7                 # once
    assert enq(ctx) == -7                                             # no field request yet
    ctx.field_enqueue((0, 0, 0), 1)                                   # a plain field request: not a known one
    ctx.field_wait()
    assert enq(ctx) == -7
    st = np.full((8, 16, 16), FREE, np.uint8)
    ctx.debug_field_load_state(st, (0, 0, 0))
    assert enq(ctx) == 0                                              # the latest request, in flight or not
    assert enq(ctx) == -7                                             # one job in flight
    assert lib.dsm_heading_wait(ctx.h, None, None, None, None) == 0
    assert lib.dsm_heading_wait(ctx.h, None, None, None, None) == -7  # nothing in flight
    ctx.field_wait()
    C = capi.DsmGainCamera
    bad = [dict(c=C(0.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)), dict(c=C(10.0, 10.0, np.nan, 5.0, 10, 10, 1.0, 1)),
           dict(c=C(10.0, 10.0, 5.0, 5.0, 0, 10, 1.0, 1)), dict(c=C(10.0, 10.0, 5.0, 5.0, 10, 65537, 1.0, 1)),
           dict(c=C(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 2)), dict(c=C(10.0, 10.0, 5.0, 5.0, 10, 10, 0.0, 1)),
           dict(c=C(10.0, 10.0, 5.0, 5.0, 10, 10, 12.81, 1)),                                  # above 128 v
           dict(n_rot=0), dict(n_rot=65), dict(r=np.where(np.arange(36).reshape(4, 9) == 3, np.inf, rot)),
           dict(k=0), dict(k=65), dict(wu=-1), dict(wf=(1 << 16) + 1), dict(n=0), dict(n=5),
           dict(o=np.array([0, 6], np.int32)), dict(o=np.array([1, 8], np.int32)),
           dict(q=np.where(np.arange(24).reshape(8, 3) == 4, np.nan, pts)),
           dict(rq=H.requests([(4, -1, 1)])), dict(rq=H.requests([(-1, -1, 1)])), dict(rq=H.requests([(0, 4, 1)])),
           dict(rq=H.requests([(0, -2, 1)])), dict(rq=H.requests([(0, -1, 5)])), dict(rq=H.requests([(0, -1, -1)]))]
    for kw in bad:
        assert enq(ctx, **kw) == -1, kw
    big = np.zeros((257, 3))
    assert enq(ctx, q=big, o=np.array([0, 257], np.int32)) == -1      # N > 256
    assert enq(ctx, q=np.zeros((16, 3)), o=np.array([0, 8, 7], np.int32), n=2, rq=H.requests([(0, -1, 1)] * 2)) == -1   # offsets fall
    assert enq(ctx, k=12) == 0 and lib.dsm_heading_wait(ctx.h, None, None, None, None) == 0   # 12 * 5 + 1 = 61 samples
    assert enq(ctx, k=13) == -1                                       # 66 samples: more than max_samples
    ctx.close()
    # the work bound: samples of (2 ceil(R / v) + 3)^3 = 259^3 voxels at R = 128 v; 124 of them pass 2^31
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(0.1, 16, 16, 8)
    ctx.views_enable(1, 1.0)
    ctx.heading_enable(64, 1 << 12)
    ctx.debug_field_load_state(np.full((8, 16, 16), FREE, np.uint8), (0, 0, 0))
    ctx.field_wait()
    far = C(10.0, 10.0, 5.0, 5.0, 10, 10, float(np.float32(12.8)), 1)
    assert H.MAX_WORK // 259 ** 3 == 123
    many = np.tile(pts, (21, 1))
    o21 = (np.arange(22) * 8).astype(np.int32)                        # trajectories of 8 points: 6 samples each at K = 1
    r21 = H.requests([(0, -1, 1)] * 21)
    assert enq(ctx, c=far, q=many, o=o21[:21], n=20, k=1, rq=r21) == 0 and lib.dsm_heading_wait(ctx.h, None, None, None, None) == 0  # 120
    assert enq(ctx, c=far, q=many, o=o21, n=21, k=1, rq=r21) == -1                                                                   # 126
    ctx.close()


# ---- the node ----
def test_node_headings_equal_the_model_and_change_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, headings() along two lines through the
    field's middle equals the model over the grid the driver dumps; clouds, PLY and PCD files equal a twin without heading
    jobs; enable_headings() before enable_known_space, headings() before any field and right after load_state return
    DSM_E_STATE."""
    cam, n = K, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = NODE_FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    r = run_driver("heading_main", str(tmp_path), cam, sc, node_args() + [1, RELOAD], tag="a", after=[pa])
    q = run_driver("heading_main", str(tmp_path), cam, sc, node_args() + [0, RELOAD], tag="b", after=[pb])
    assert r.i() == -7 and r.i() == 0 and r.i() == -7
    planned = 0
    for t in range(n):
        rc, ub = r.i(), r.i()
        max_range = float(r.take(np.float32, 1)[0])
        Ks, origin = r.i(), r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        pts, ofs, rot = r.lst(np.float64).reshape(-1, 3), r.lst(np.int32), r.lst(np.float64).reshape(-1, 9)
        req = r.lst(H.REQUEST_DTYPE)
        info = r.take(np.uint8, H.INFO_DTYPE.itemsize).view(H.INFO_DTYPE)[0].copy()
        recs, samples, counts = r.lst(H.RECORD_DTYPE), r.lst(H.SAMPLE_DTYPE), r.lst(H.COUNT_DTYPE)
        after_load = r.i()
        twin_clouds(r, q, f"message {t}")
        assert rc == 0, f"message {t}: {rc}"
        gc = G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, max_range, ub)
        same((info, recs, samples, counts.reshape(-1, len(rot))), H.job(state, origin, voxel, gc, rot, Ks, pts, ofs, req, 2, 3),
             f"message {t}", NAMES)
        planned += int((recs["score"] > 0).any())
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: headings() after load_state"
    assert planned > 0
    twin_node_tail(r, q, pa, pb)
