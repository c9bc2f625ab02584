"""GPU parity tests proper: the CUDA path, called through the C ABI (include/dsm.h), against the
oracle on the same seeded inputs.  Bar: labels + clustering state bit-exact, surfel geometry
within 1e-4 (norm-based), integer fields exact."""
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import bits_equal_nan, check_seeds, check_surfels, compact_like_caller, oracle_for

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    from densesurfelmapping_b200 import capi as m
    m.load_library()  # raises if the CUDA extension was not built: no fallback
    return m


def _stream(capi, cam, n_frames, flat=False, ref_div=2):
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=200000)
    orc = oracle_for(cam)
    pool_g = np.zeros(0, SURFEL_DTYPE)
    pool_o = np.zeros(0, SURFEL_DTYPE)
    for t in range(n_frames):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, t, pose, flat=flat)
        lo, no = orc.fuse(t // ref_div, gray, depth, pose, pool_o)
        lg, ng = ctx.fuse_frame(t // ref_div, gray, depth, pose, pool_g)
        lab_o, lab_g = orc.labels(), ctx.labels()
        nbad = int((lab_o != lab_g).sum())
        assert nbad == 0, f"frame {t}: {nbad} label mismatches (first at {np.argwhere(lab_o != lab_g)[:4].tolist()})"
        check_seeds(ctx.seeds(), orc.seeds())
        assert ctx.invariant_violations() == 0
        check_surfels(lg, lo, f"frame {t} local")
        check_surfels(ng, no, f"frame {t} new")
        # carry the ORACLE's pool into both so that one tolerance-sized drift cannot compound
        pool_o = compact_like_caller(lo, no)
        pool_g = pool_o.copy()
    ctx.close()


def test_stage_by_stage_vga(capi):
    """Localises a mismatch to one pass: after each assign / update the labels and the
    clustering state must equal the restatement's."""
    import pyoracle
    cam = synth.VGA
    gray, depth = synth.make_frame(cam, 0)
    ro = pyoracle.Restatement(cam)
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=16)
    pose = synth.identity_pose()
    ctx.batch_upload([0], gray[None], depth[None], pose[None], np.zeros(0, SURFEL_DTYPE), [0, 0])
    # (kernels to run, oracle iterations, last-with-update); tile schedule: seed_init, then (assign, gather, newton) x 3
    stages = [(2, 1, False), (4, 1, True), (5, 2, False), (7, 2, True), (8, 3, False), (10, 3, True)]
    for nk, iters, upd in stages:
        ctx.debug_stop_after(nk)
        ctx.batch_run()
        ctx.sync()
        lab_o, seeds_o = ro.debug_iters(gray, depth, iters, upd)
        lab_g, seeds_g = ctx.labels(), ctx.seeds()
        nbad = int((lab_o != lab_g).sum())
        assert nbad == 0, f"after {nk} kernels: {nbad} label mismatches, first {np.argwhere(lab_o != lab_g)[:4].tolist()}"
        for f in ("x", "y", "mean_intensity", "mean_depth"):
            bad = np.nonzero(~bits_equal_nan(seeds_g[f], seeds_o[f]))[0]
            assert len(bad) == 0, f"after {nk} kernels: seed.{f} differs at {bad[:6]}: {seeds_g[f][bad[:6]]} vs {seeds_o[f][bad[:6]]}"
        bad = np.nonzero(seeds_g["stable"] != seeds_o["stable"])[0]
        assert len(bad) == 0, f"after {nk} kernels: stable differs at {bad[:8]}"
    ctx.debug_stop_after(0)
    ctx.close()


def test_single_frame_vga_identity(capi):
    """BASELINE config 1: one 640x480 frame, identity pose, empty pool then the same frame again."""
    cam = synth.VGA
    gray, depth = synth.make_frame(cam, 0)
    pose = synth.identity_pose()
    orc = oracle_for(cam)
    ff = capi.FusionFunctions()
    ff.initialize(cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)
    lo, no = orc.fuse(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    lg, ng = ff.fuse_initialize_map(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    assert (orc.labels() == ff._ctx.labels()).all()
    check_surfels(ng, no, "initialise")
    lo2, no2 = orc.fuse(1, gray, depth, pose, no)
    lg2, ng2 = ff.fuse_initialize_map(1, gray, depth, pose, no)
    assert (orc.labels() == ff._ctx.labels()).all()
    check_seeds(ff._ctx.seeds(), orc.seeds())
    check_surfels(lg2, lo2, "fuse")
    check_surfels(ng2, no2, "new after fuse")
    assert (lg2["update_times"] > 1).sum() > 100  # the pure-fuse case really fused


def test_stream_kitti(capi):
    """BASELINE config 2 shape: 1226x370 stream with a carried pool (fuse + kill + initialise)."""
    _stream(capi, synth.KITTI, 4)


def test_stream_kitti_flat(capi):
    """Noise-free piecewise-constant scene: the summation-order-sensitive case (SURVEY H2) and
    the NaN-normal seeds (H6-iii)."""
    _stream(capi, synth.KITTI, 3, flat=True)


def test_stream_vga_flat(capi):
    _stream(capi, synth.VGA, 3, flat=True)


def test_stream_hd(capi):
    """BASELINE config 5 shape (1280x720)."""
    _stream(capi, synth.HD, 2)


def test_kitti00_shape(capi):
    """1241x376 (W%8 == 1, H%8 == 0): the real KITTI-00 frame size."""
    _stream(capi, synth.KITTI00, 2)


def test_batch_matches_per_frame(capi):
    """BASELINE config 3 shape: a batch of independent frames, each with its own pool slice."""
    cam = synth.KITTI
    B = 5
    orc = oracle_for(cam)
    grays, depths, poses, refs, pools = [], [], [], [], []
    for b in range(B):
        pose0 = synth.pose_stream(b)
        g0, d0 = synth.make_frame(cam, 100 + b, pose0)
        _, seeded = orc.fuse(0, g0, d0, pose0, np.zeros(0, SURFEL_DTYPE))  # predecessor view -> pool
        pose1 = synth.pose_stream(b + 1)
        g1, d1 = synth.make_frame(cam, 200 + b, pose1)
        grays.append(g1), depths.append(d1), poses.append(pose1), refs.append(b % 3), pools.append(seeded if b != 2 else seeded[:0])
    offsets = np.concatenate([[0], np.cumsum([len(p) for p in pools])]).astype(np.int32)
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=int(offsets[-1]) + 8)
    local, news = ctx.fuse_batch(refs, np.stack(grays), np.stack(depths), np.stack(poses), np.concatenate(pools), offsets)
    for b in range(B):
        lo, no = orc.fuse(refs[b], grays[b], depths[b], poses[b], pools[b])
        assert (orc.labels() == ctx.labels(b)).all(), f"batch frame {b} labels"
        check_seeds(ctx.seeds(b), orc.seeds())
        check_surfels(local[offsets[b]:offsets[b + 1]], lo, f"batch frame {b} local")
        check_surfels(news[b], no, f"batch frame {b} new")
    ctx.close()


def test_concurrent_sub_batches_do_not_change_results(capi):
    """dsm_set_concurrency: a resident batch as 1, 2, 3 or 4 groups of frames on concurrent streams gives byte-identical
    outputs (frames are independent); two frames of the batch are also checked against the reference."""
    cam = synth.Camera(132, 100, 60.0, 60.0, 65.5, 49.5, 0.5, 30.0)
    B = 9
    frames = [synth.make_frame(cam, 300 + i, synth.pose_stream(i)) for i in range(B)]
    g, d = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    p = np.stack([synth.pose_stream(i) for i in range(B)])
    ctx = capi.Context(cam, max_batch=B, max_local_surfels=8192)
    _, pools = ctx.fuse_batch([0] * B, g, d, p, np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    ofs = np.concatenate([[0], np.cumsum([len(x) for x in pools])]).astype(np.int32)
    p2 = np.stack([synth.pose_stream(i + 1) for i in range(B)])
    outs = []
    for parts in (1, 2, 3, 4, 2):
        ctx.set_concurrency(parts)
        ctx.batch_upload([1] * B, g, d, p2, np.concatenate(pools), ofs)
        ctx.batch_run()
        local, news = ctx.batch_download()
        outs.append((local.tobytes(), [n.tobytes() for n in news], [ctx.labels(b).tobytes() for b in (0, B - 1)]))
    assert all(o == outs[0] for o in outs[1:])
    with pytest.raises(Exception):
        ctx.set_concurrency(5)
    orc = oracle_for(cam)
    for b in (0, B - 1):
        lo, no = orc.fuse(1, g[b], d[b], p2[b], pools[b])
        assert (orc.labels() == ctx.labels(b)).all()
        check_surfels(local[ofs[b]:ofs[b + 1]], lo, f"frame {b} local")
        check_surfels(news[b], no, f"frame {b} new")
    ctx.close()


def test_pitched_input_and_errors(capi):
    import ctypes
    cam = synth.VGA
    gray, depth = synth.make_frame(cam, 7)
    gp = np.full((cam.height, cam.width + 24), 0xEE, np.uint8)  # pad columns hold garbage the call must not read
    dp = np.full((cam.height, cam.width + 8), 99.0, np.float32)
    gp[:, :cam.width] = gray
    dp[:, :cam.width] = depth
    pose = synth.identity_pose()

    def fuse_padded(ctx, local, new, cap):
        n = ctypes.c_int(-1)
        rc = ctx.lib.dsm_fuse_frame(ctx.h, 0, gp.ctypes.data, gp.strides[0], dp.ctypes.data, dp.strides[0], pose.ctypes.data,
                                    local.ctypes.data if len(local) else None, len(local), new.ctypes.data, cap, ctypes.byref(n))
        assert rc == 0
        return n.value

    ctx = capi.Context(cam, max_batch=1, max_local_surfels=16)
    new = np.zeros(ctx.S, SURFEL_DTYPE)
    n = fuse_padded(ctx, np.zeros(0, SURFEL_DTYPE), new, ctx.S)
    _, want = oracle_for(cam).fuse(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    check_surfels(new[:n], want, "pitched")
    pool = new[:n // 2].copy()  # covers part of the frame: the next fuse both fuses and initialises
    # capacity error: more local surfels than the context was created for
    with pytest.raises(capi.DsmError) as ei:
        ctx.fuse_frame(0, gray, depth, pose, np.zeros(17, SURFEL_DTYPE))
    assert ei.value.code == -6
    ctx.close()
    # on a non-empty pool, padded rows give byte for byte what packed rows give; with new_cap below the count exactly
    # new_cap surfels are written, the rest of the buffer is untouched and *n_new is the full count
    for max_batch in (1, 8):
        ctx = capi.Context(cam, max_batch=max_batch, max_local_surfels=1 << 16)
        want_local, want_new = ctx.fuse_frame(0, gray, depth, pose, pool)
        assert (want_local["update_times"] > 1).any() and len(want_new) > 1
        want_labels, want_seeds = ctx.labels().tobytes(), ctx.seeds().tobytes()
        local, new = pool.copy(), np.zeros(ctx.S, SURFEL_DTYPE)
        assert fuse_padded(ctx, local, new, ctx.S) == len(want_new)
        assert local.tobytes() == want_local.tobytes() and new[:len(want_new)].tobytes() == want_new.tobytes()
        assert ctx.labels().tobytes() == want_labels and ctx.seeds().tobytes() == want_seeds
        cap = len(want_new) // 2
        local = pool.copy()
        new = np.frombuffer(b"\xa5" * (ctx.S * SURFEL_DTYPE.itemsize), SURFEL_DTYPE).copy()
        assert fuse_padded(ctx, local, new, cap) == len(want_new)
        assert local.tobytes() == want_local.tobytes() and new[:cap].tobytes() == want_new[:cap].tobytes()
        assert new[cap:].tobytes() == b"\xa5" * ((ctx.S - cap) * SURFEL_DTYPE.itemsize)
        ctx.close()
    # shape error: W%8 > 4 is undefined behaviour in the reference (fusion_functions.cpp:408-451)
    bad = synth.Camera(645, 480, 525.0, 525.0, 319.5, 239.5, 0.5, 30.0)
    with pytest.raises(capi.DsmError) as ei:
        capi.Context(bad)
    assert ei.value.code == -2


@pytest.mark.parametrize("case", ["no_depth", "constant", "binary_noise_holes", "checker_steps", "tiny_depths"])
def test_adversarial_small_frames(capi, case):
    """Edge inputs on an odd shape (W%8 == 4, H%8 == 2): no depth at all (only the no-depth cost path),
    a constant image (every seed goes stable after the first update, so EVERY pixel of passes 2-3 goes
    through the deferred list / k_relax), salt-and-pepper gray with 50 % holes (maximal label churn),
    a checkerboard with depth steps (plane fits rejected / NaN normals), and depths around the three
    validity thresholds 0.01 / 0.05 / 0.1.  (Valid depths stay >= 0.02 m: below that every candidate's
    depth cost exceeds the reference's 1e6 sentinel, its argmin index stays -1 and it writes out of
    bounds, fusion_functions.cpp:408-451 -- undefined there, see DESIGN.md 1.3.)"""
    cam = synth.Camera(324, 242, 260.0, 260.0, 161.5, 120.5, 0.5, 30.0)
    H, W = cam.height, cam.width
    rng = np.random.RandomState(99)
    yy, xx = np.mgrid[0:H, 0:W]
    if case == "no_depth":
        gray = rng.randint(0, 256, (H, W)).astype(np.uint8)
        depth = np.zeros((H, W), np.float32)
    elif case == "constant":
        gray = np.full((H, W), 77, np.uint8)
        depth = np.full((H, W), 3.0, np.float32)
    elif case == "binary_noise_holes":
        gray = (rng.randint(0, 2, (H, W)) * 255).astype(np.uint8)
        depth = rng.uniform(0.5, 20.0, (H, W)).astype(np.float32)
        depth[rng.rand(H, W) < 0.5] = 0
    elif case == "checker_steps":
        gray = (((xx // 8 + yy // 8) % 2) * 200 + 20).astype(np.uint8)
        depth = (2.0 + 3.0 * ((xx // 16 + yy // 16) % 2)).astype(np.float32)
    else:
        gray = (xx % 256).astype(np.uint8)
        depth = rng.choice(np.array([0.0, 0.009, 0.021, 0.049, 0.051, 0.099, 0.101, 0.5, 2.0], np.float32), size=(H, W))
    orc = oracle_for(cam)
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=20000)
    pose = synth.pose_stream(1)
    pool = np.zeros(0, SURFEL_DTYPE)
    for rep in range(2):  # second pass fuses against the surfels of the first
        lo, no = orc.fuse(rep, gray, depth, pose, pool)
        lg, ng = ctx.fuse_frame(rep, gray, depth, pose, pool)
        nbad = int((orc.labels() != ctx.labels()).sum())
        assert nbad == 0, f"{case} rep {rep}: {nbad} label mismatches"
        check_seeds(ctx.seeds(), orc.seeds())
        assert ctx.invariant_violations() == 0
        check_surfels(lg, lo, f"{case} local")
        check_surfels(ng, no, f"{case} new")
        pool = compact_like_caller(lo, no)
    ctx.close()


def test_async_batch_double_buffering(capi):
    """dsm_fuse_batch_async + dsm_batch_wait on two alternating contexts gives the same bytes as the
    synchronous dsm_fuse_batch."""
    cam = synth.VGA
    B = 3
    frames = [synth.make_frame(cam, 700 + b, synth.pose_stream(b)) for b in range(B)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames])
    poses = np.stack([synth.pose_stream(b) for b in range(B)])
    refs = np.zeros(B, np.int32)
    ofs = np.zeros(B + 1, np.int32)
    ctxs = [capi.Context(cam, max_batch=B, max_local_surfels=64) for _ in range(2)]
    S = ctxs[0].S
    want_local, want_new = ctxs[0].fuse_batch(refs, gray, depth, poses, np.zeros(0, SURFEL_DTYPE), ofs)
    outs = []
    for k in range(4):
        c = ctxs[k & 1]
        new = np.zeros((B, S), SURFEL_DTYPE)
        cnt = np.zeros(B, np.int32)
        assert c.lib.dsm_batch_wait(c.h) == 0
        rc = c.lib.dsm_fuse_batch_async(c.h, B, refs.ctypes.data, gray.ctypes.data, depth.ctypes.data, poses.ctypes.data,
                                        None, ofs.ctypes.data, new.ctypes.data, cnt.ctypes.data)
        assert rc == 0
        outs.append((c, new, cnt))
    for c, new, cnt in outs:
        assert c.lib.dsm_batch_wait(c.h) == 0
        for b in range(B):
            assert cnt[b] == len(want_new[b]) and new[b, :cnt[b]].tobytes() == want_new[b].tobytes()
    for c in ctxs:
        c.close()


def test_random_small_images(capi):
    """40 random 64x48 frames inside the input domain (noise, salt-and-pepper, ramps, holes, exact depth
    ties): labels bit-exact, clustering state bit-exact, plane fits within tolerance."""
    cam = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
    orc = oracle_for(cam)
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=64)
    yy, xx = np.mgrid[0:48, 0:64]
    pose = synth.identity_pose()
    for seed in range(40):
        rng = np.random.RandomState(seed)
        mode = seed % 3
        if mode == 0:
            gray = rng.randint(0, 256, (48, 64)).astype(np.uint8)
        elif mode == 1:
            gray = (rng.randint(0, 2, (48, 64)) * 255).astype(np.uint8)
        else:
            gray = ((xx * 3 + yy * 2 + rng.randint(0, 4, (48, 64))) % 256).astype(np.uint8)
        depth = rng.uniform(0.02, 25.0, (48, 64)).astype(np.float32)
        if seed % 2:
            depth[rng.rand(48, 64) < 0.4] = 0
        if seed % 5 == 0:
            depth = np.round(depth)
        _, no = orc.fuse(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
        _, ng = ctx.fuse_frame(0, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
        nbad = int((orc.labels() != ctx.labels()).sum())
        assert nbad == 0, f"image {seed}: {nbad} label mismatches"
        check_seeds(ctx.seeds(), orc.seeds())
        check_surfels(ng, no, f"image {seed} new")
    ctx.close()


def test_rgbd_constant_set_hd(capi):
    """BASELINE configs[4] flavour: 1280x720 with the reference's second constant set (fusion_functions.h:17-21,
    selected at run time with dsm_set_constants) against the reference source compiled with those #defines."""
    import pyoracle
    cam = synth.Camera(1280, 720, 720.0, 720.0, 639.5, 359.5, 0.3, 8.0)
    have_ref = os.path.exists(os.path.join(pyoracle.REFDIR, "libdsm_ref_serial_rgbd.so"))
    orc = pyoracle.RefSerialRGBD(cam) if have_ref else pyoracle.Restatement(cam, pyoracle.CONSTANTS_RGBD)
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=1 << 17)
    ctx.set_constants(capi.CONSTANTS_RGBD)
    pool_o = pool_g = np.zeros(0, SURFEL_DTYPE)
    for t in range(2):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 700 + t, pose)
        depth = (depth * np.float32(0.2)).astype(np.float32)  # indoor range: the RGBD set assumes metres of a room
        lo, no = orc.fuse(t, gray, depth, pose, pool_o)
        lg, ng = ctx.fuse_frame(t, gray, depth, pose, pool_g)
        assert (ctx.labels() == orc.labels()).all()
        check_seeds(ctx.seeds(), orc.seeds())
        check_surfels(lg, lo, "local")
        check_surfels(ng, no, "new")
        assert ctx.invariant_violations() == 0
        pool_o = compact_like_caller(lo, no)
        pool_g = compact_like_caller(lg, ng)
    ctx.set_constants(capi.CONSTANTS_DRIVE)  # and back: the drive set must give something else on this data
    _, nd = ctx.fuse_frame(5, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    _, nr = orc.fuse(5, gray, depth, pose, np.zeros(0, SURFEL_DTYPE))
    assert len(nd) != len(nr) or not np.array_equal(nd["pz"], nr["pz"])
    ctx.close()
