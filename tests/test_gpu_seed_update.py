"""GPU tests: the superpixel clustering state after every pass, bit for bit against the restatement, on the inputs
that reach every branch of the Huber-Newton seed update (tests/seed_update_inputs.py, reach proven on the host by
tests/test_seed_update_paths.py), over the seed-tile remainders, both constant sets and several batch slots; the whole seed state of every frame of
a batch run as concurrent sub-batches; and the plane fit of an input that reaches the plane solver's second phase."""
import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from seed_update_inputs import cam_of, checker_frame, far_frame, plane_frame, scene_frame
from util import bits_equal_nan, check_seeds, check_surfels, oracle_for

pytestmark = pytest.mark.gpu

# spw % 8 in {0, 1, 3, 4, 6}, sph % 4 in {0, 1, 2, 3}, every W % 8 and H % 8 in 0..4
SHAPES = [(64, 48), (97, 66), (130, 83), (244, 100), (160, 124), (139, 76), (324, 242), (1226, 370), (1241, 376), (1280, 720)]
# (kernels to run, restatement passes, last pass with its update): seed init, then (assign, gather, Newton) x 3
STOPS = [(2, 1, False), (4, 1, True), (5, 2, False), (7, 2, True), (8, 3, False), (10, 3, True)]


@pytest.fixture(scope="module")
def capi():
    from densesurfelmapping_b200 import capi as m
    m.load_library()  # raises if the CUDA extension was not built: no fallback
    return m


def batch_frames(w, h, rgbd):
    """The large-depth frame in slot 0, the checkerboard and a scene frame in slots 1 and 2, and the three again in
    slots 3 - 5: every frame runs in an early and in a later slot, the large-depth one in slot 0."""
    g0, d0 = scene_frame(cam_of(w, h), 40 + w % 7)
    if rgbd:
        d0 = (d0 * np.float32(0.15)).astype(np.float32)  # metres of a room
    frames = [far_frame(w, h), checker_frame(w, h), (g0, d0)]
    return frames + frames


def compare(ctx, b, lab_o, seeds_o, what):
    lab_g, seeds_g = ctx.labels(b), ctx.seeds(b)
    nbad = int((lab_o != lab_g).sum())
    assert nbad == 0, f"{what}: {nbad} label mismatches, first {np.argwhere(lab_o != lab_g)[:4].tolist()}"
    for f in ("x", "y", "mean_intensity", "mean_depth"):
        bad = np.nonzero(~bits_equal_nan(seeds_g[f], seeds_o[f]))[0]
        assert len(bad) == 0, f"{what}: seed.{f} differs at {bad[:6]}: {seeds_g[f][bad[:6]]} vs {seeds_o[f][bad[:6]]}"
    bad = np.nonzero(seeds_g["stable"] != seeds_o["stable"])[0]
    assert len(bad) == 0, f"{what}: seed.stable differs at {bad[:8]}"


@pytest.mark.parametrize("rgbd", [False, True], ids=["drive", "rgbd"])
@pytest.mark.parametrize("w,h", SHAPES)
def test_every_pass_is_bit_exact(capi, w, h, rgbd):
    """After each assign and each seed update: labels and x, y, mean_intensity, mean_depth, stable equal the
    restatement's bit for bit (NaN == NaN), for every frame of a 6-frame batch; no invariant is violated."""
    cam = cam_of(w, h)
    consts = pyoracle.CONSTANTS_RGBD if rgbd else pyoracle.CONSTANTS_DRIVE
    frames = batch_frames(w, h, rgbd)
    B = len(frames)
    ro = pyoracle.Restatement(cam, consts)
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=16)
    ctx.set_constants(capi.CONSTANTS_RGBD if rgbd else capi.CONSTANTS_DRIVE)
    gray, depth = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    ctx.batch_upload([0] * B, gray, depth, np.stack([synth.identity_pose()] * B), np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    try:
        for nk, iters, upd in STOPS:
            ctx.debug_stop_after(nk)
            ctx.batch_run()
            ctx.sync()
            assert ctx.invariant_violations() == 0, f"after {nk} kernels"
            for b in range(B // 2):
                lab_o, seeds_o = ro.debug_iters(gray[b], depth[b], iters, upd)
                for slot in (b, b + B // 2):  # the same frame in both of its slots
                    compare(ctx, slot, lab_o, seeds_o, f"{w}x{h} slot {slot} after {nk} kernels")
    finally:
        ctx.debug_stop_after(0)
        ctx.close()


@pytest.mark.parametrize("parts", [2, 3, 4])
def test_concurrent_sub_batches_give_every_frame_its_seeds(capi, parts):
    """A 9-frame batch split into concurrent sub-batches (dsm_set_concurrency): every frame's labels equal the
    oracle's and its seeds pass check_seeds (clustering state bit-exact, plane fits within tolerance)."""
    cam = synth.Camera(324, 242, 260.0, 260.0, 161.5, 120.5, 0.5, 30.0)
    B = 9
    frames = [synth.make_frame(cam, 500 + i, synth.pose_stream(i)) for i in range(B)]
    g, d = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    p = np.stack([synth.pose_stream(i) for i in range(B)])
    orc = oracle_for(cam)
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=64)
    ctx.set_concurrency(parts)
    ctx.fuse_batch([0] * B, g, d, p, np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    assert ctx.invariant_violations() == 0
    for b in range(B):
        orc.fuse(0, g[b], d[b], p[b], np.zeros(0, SURFEL_DTYPE))
        assert (orc.labels() == ctx.labels(b)).all(), f"frame {b} labels"
        check_seeds(ctx.seeds(b), orc.seeds())
    ctx.close()


def test_plane_solver_second_phase(capi):
    """The plane input (tests/seed_update_inputs.py): at 139 x 76, 41 seeds go through k_gn_solve's phase B and the
    first 128-seed block's point lists overflow its shared staging (proven on the host by test_seed_update_paths.py).
    Labels and the clustering state bit-exact, plane fits within tolerance, as a single frame and in slot 2 of a batch.
    (The input is noise about a surface, where the reference's damped fit shrinks (n, b) towards 0 and the direction
    of the normal is only as stable as the rounding allows -- DESIGN.md 1.3; the committed frame is one where it is.)"""
    w, h = 139, 76
    cam = cam_of(w, h)
    g, d = plane_frame(w, h)
    orc = oracle_for(cam)
    _, no = orc.fuse(0, g, d, synth.identity_pose(), np.zeros(0, SURFEL_DTYPE))
    lab_o, seeds_o = orc.labels(), orc.seeds()
    ctx = capi.Context(cam, max_batch=3, max_local_surfels=64)
    _, ng = ctx.fuse_frame(0, g, d, synth.identity_pose(), np.zeros(0, SURFEL_DTYPE))
    assert (ctx.labels() == lab_o).all()
    check_seeds(ctx.seeds(), seeds_o)
    check_surfels(ng, no, "plane frame new")
    assert ctx.invariant_violations() == 0
    frames = [far_frame(w, h), checker_frame(w, h), (g, d)]
    _, news = ctx.fuse_batch([0] * 3, np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]),
                             np.stack([synth.identity_pose()] * 3), np.zeros(0, SURFEL_DTYPE), np.zeros(4, np.int32))
    assert (ctx.labels(2) == lab_o).all()
    check_seeds(ctx.seeds(2), seeds_o)
    check_surfels(news[2], no, "plane frame new, batch slot 2")
    assert ctx.invariant_violations() == 0
    ctx.close()
