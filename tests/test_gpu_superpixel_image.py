"""dsm_frame_superpixel_image on the H100: the superpixel normal image of FusionFunctions::debug_show
(fusion_functions.cpp:977-1006) from the frame slots of every entry point that takes images.

Given the context's own labels and seeds (dsm_get_labels / dsm_get_seeds of the same slot) the image equals the numpy
restatement the CPU suite pins, and the reference's own debug_show fed those arrays, byte for byte.  Against the
reference's whole pipeline on the same frame the black boundary pixels are exact and colours differ by at most 1.
Also: the error returns, untouched padding bytes of a pitched output, no effect on the pool, and the C++ helpers."""
import ctypes
import struct
import subprocess

import numpy as np
import pytest

import pyoracle
import pyoracle_show
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from test_cpp_adapter import build_adapter
from test_refmap import CAM

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -7


def frames(cam, n, seed, flat=False):
    out = []
    for t in range(n):
        pose = synth.pose_stream(seed + t)
        g, d = synth.make_frame(cam, seed + t, pose, flat=flat)
        out.append((pose, g, d))
    return out


def pipeline(cam, gray, depth):
    """labels and seeds of the reference's whole superpixel stage on this frame (the serial reference where it is built,
    else the restatement, which is byte-identical to it)"""
    orc = pyoracle.RefSerial(cam) if pyoracle.have_reference() else pyoracle.Restatement(cam)
    labels, seeds = orc.superpixels(gray, depth)
    orc.close()
    return labels, seeds


def check_image(ctx, frame, slot, gray, depth, what):
    cam = ctx.cam
    got = ctx.superpixel_image(frame)
    assert got.shape == (cam.height, cam.width, 3) and got.dtype == np.uint8, what
    # 1. the context's own state: byte-identical to debug_show over dsm_get_labels + dsm_get_seeds of the slot
    labels, seeds = ctx.labels(slot), ctx.seeds(slot)
    want = pyoracle_show.superpixel_image(labels, seeds)
    assert got.tobytes() == want.tobytes(), f"{what}: {(got != want).any(2).sum()} pixels differ from the restatement"
    if pyoracle_show.have_ref_show():
        m = pyoracle_show.RefShow(cam)
        assert got.tobytes() == m.debug_show(labels, seeds).tobytes(), f"{what}: differs from the reference's debug_show"
        m.close()
    # 2. the reference's whole pipeline on this frame: same labels, hence the same black boundary; colours within 1
    rl, rs = pipeline(cam, gray, depth)
    assert (labels == rl).all(), f"{what}: slot {slot} does not hold this frame's labels"
    ref = pyoracle_show.superpixel_image(rl, rs)
    edge = np.zeros(rl.shape, bool)
    edge[:, :-1] |= rl[:, 1:] != rl[:, :-1]
    edge[:-1, :] |= rl[1:, :] != rl[:-1, :]
    assert (got[edge] == 0).all(), what
    diff = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    assert diff.max() <= 1, f"{what}: colour off by {diff.max()}"
    return got


@pytest.mark.parametrize("cam", [synth.VGA, synth.KITTI], ids=["vga", "kitti"])
def test_after_fuse_frame_resident_both_slots(cam):
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=200000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for t, (pose, g, d) in enumerate(frames(cam, 3, 40)):   # frame slots 0, 1, 0
        ctx.fuse_frame_resident(t, g, d, pose)
        check_image(ctx, 0, t % 2, g, d, f"resident frame {t}")
    ctx.close()


def test_after_fuse_stream_resident_both_halves():
    cam = synth.VGA
    ctx = capi.Context(cam, max_batch=8, max_local_surfels=400000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for run in range(2):   # two runs of 4 frames: slots 0..3, then 4..7
        fr = frames(cam, 4, 60 + 4 * run, flat=(run == 1))
        ctx.fuse_stream_resident(np.arange(4) + 4 * run, np.stack([g for _, g, _ in fr]), np.stack([d for _, _, d in fr]),
                                 np.stack([p for p, _, _ in fr]))
        for b, (_, g, d) in enumerate(fr):
            check_image(ctx, b, 4 * run + b, g, d, f"stream run {run} frame {b}")
    ctx.close()


def batch_args(cam, n, seed, flat=False):
    fr = frames(cam, n, seed, flat)
    return (np.arange(n, dtype=np.int32), np.ascontiguousarray(np.stack([g for _, g, _ in fr])),
            np.ascontiguousarray(np.stack([d for _, _, d in fr])), np.ascontiguousarray(np.stack([p for p, _, _ in fr])))


def test_after_batch_calls():
    cam = synth.KITTI
    n = 4
    ref, g, d, p = batch_args(cam, n, 80)
    ctx = capi.Context(cam, max_batch=n, max_local_surfels=1000)
    L, S = ctx.lib, ctx.S
    ofs = np.zeros(n + 1, np.int32)
    new = np.zeros(n * S, SURFEL_DTYPE)
    cnt = np.zeros(n, np.int32)
    buf = np.zeros((cam.height, 3 * cam.width), np.uint8)
    # dsm_batch_upload: the frames are there, but their schedule has not run
    ctx.batch_upload(ref, g, d, p, np.zeros(0, SURFEL_DTYPE), ofs)
    assert L.dsm_frame_superpixel_image(ctx.h, 1, buf.ctypes.data, buf.strides[0]) == E_STATE
    ctx._ck(L.dsm_batch_run(ctx.h))
    check_image(ctx, 1, 1, g[1], d[1], "dsm_batch_upload + dsm_batch_run frame 1")
    ctx._ck(L.dsm_fuse_batch(ctx.h, n, ref.ctypes.data, g.ctypes.data, d.ctypes.data, p.ctypes.data, None,
                             ofs.ctypes.data, new.ctypes.data, cnt.ctypes.data))
    check_image(ctx, 2, 2, g[2], d[2], "dsm_fuse_batch frame 2")
    # asynchronous batch (chunks on their own streams), image asked for before dsm_batch_wait
    ref2, g2, d2, p2 = batch_args(cam, n, 90, flat=True)
    ctx._ck(L.dsm_fuse_batch_async(ctx.h, n, ref2.ctypes.data, g2.ctypes.data, d2.ctypes.data, p2.ctypes.data, None,
                                   ofs.ctypes.data, new.ctypes.data, cnt.ctypes.data))
    check_image(ctx, 3, 3, g2[3], d2[3], "dsm_fuse_batch_async frame 3")
    ctx._ck(L.dsm_batch_wait(ctx.h))
    check_image(ctx, 0, 0, g2[0], d2[0], "dsm_fuse_batch_async frame 0")
    ctx.close()


def fuse_frame(ctx, pose, g, d):
    n = ctypes.c_int(0)
    new = np.zeros(ctx.S, SURFEL_DTYPE)
    pose = np.ascontiguousarray(pose, np.float32)
    return ctx.lib.dsm_fuse_frame(ctx.h, 0, g.ctypes.data, g.strides[0], d.ctypes.data, d.strides[0], pose.ctypes.data,
                                  None, 0, new.ctypes.data, ctx.S, ctypes.byref(n))


def test_after_fuse_frame_errors_and_padding():
    cam = CAM
    W, H = cam.width, cam.height
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=100000)
    L = ctx.lib
    buf = np.zeros((H, 3 * W), np.uint8)
    assert L.dsm_frame_superpixel_image(ctx.h, 0, buf.ctypes.data, buf.strides[0]) == E_STATE   # no call took images yet
    (pose, g, d), (pose2, g2, d2) = frames(cam, 2, 120, flat=True)
    # a run cut short before the plane fit: no image; through the plane fit: the image of that state
    ctx.debug_stop_after(5)
    assert fuse_frame(ctx, pose, g, d) == 0
    assert L.dsm_frame_superpixel_image(ctx.h, 0, buf.ctypes.data, buf.strides[0]) == E_STATE
    ctx.debug_stop_after(12)
    assert fuse_frame(ctx, pose, g, d) == 0
    check_image(ctx, 0, 0, g, d, "dsm_fuse_frame stopped after the plane fit")
    ctx.debug_stop_after(0)
    assert fuse_frame(ctx, pose2, g2, d2) == 0
    full = check_image(ctx, 0, 0, g2, d2, "dsm_fuse_frame")
    # pitched output: the padding bytes keep what the caller had there
    pitch = 3 * W + 29
    padded = (np.arange(H * pitch, dtype=np.int64) * 7 % 251).astype(np.uint8).reshape(H, pitch)
    before = padded.copy()
    assert L.dsm_frame_superpixel_image(ctx.h, 0, padded.ctypes.data, pitch) == 0
    assert padded[:, :3 * W].tobytes() == full.tobytes()
    assert padded[:, 3 * W:].tobytes() == before[:, 3 * W:].tobytes()
    assert ctx.superpixel_image(0, pitch=pitch).tobytes() == full.tobytes()
    # invalid arguments
    for frame, ptr, pt in ((1, buf.ctypes.data, 3 * W), (-1, buf.ctypes.data, 3 * W), (0, None, 3 * W),
                           (0, buf.ctypes.data, 3 * W - 1), (0, buf.ctypes.data, 0)):
        assert L.dsm_frame_superpixel_image(ctx.h, frame, ptr, pt) == E_INVALID
    assert L.dsm_frame_superpixel_image(None, 0, buf.ctypes.data, 3 * W) == E_INVALID
    with pytest.raises(capi.DsmError):
        ctx.superpixel_image(2)
    ctx.close()


def test_no_side_effects_on_the_stream():
    """Two identical resident streams, one asking for the image between frames: the pools end identical, and so do the
    labels and seeds of the last frame."""
    cam = synth.VGA
    fr = frames(cam, 5, 300)
    ctxs = [capi.Context(cam, max_batch=8, max_local_surfels=400000) for _ in range(2)]
    for k, ctx in enumerate(ctxs):
        ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
        for t, (pose, g, d) in enumerate(fr[:3]):
            ctx.fuse_frame_resident(t, g, d, pose)
            if k == 1:
                ctx.superpixel_image(0)
        run = fr[3:]
        ctx.fuse_stream_resident(np.arange(3, 5), np.stack([g for _, g, _ in run]), np.stack([d for _, _, d in run]),
                                 np.stack([p for p, _, _ in run]))
        if k == 1:
            ctx.superpixel_image(0), ctx.superpixel_image(1)
    a, b = ctxs
    assert a.pool_download().tobytes() == b.pool_download().tobytes()
    for slot in (0, 1, 4, 5):   # the single-frame slots 0 / 4, and the stream's half (its 4th run -> the second half)
        assert a.labels(slot).tobytes() == b.labels(slot).tobytes() and a.seeds(slot).tobytes() == b.seeds(slot).tobytes()
    for c in ctxs:
        c.close()


def test_cpp_helpers(tmp_path):
    cam = CAM
    W, H = cam.width, cam.height
    exe = build_adapter("superpixel_image_main")
    fr = frames(cam, 3, 200)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<i", len(fr)))
        for t, (pose, g, d) in enumerate(fr):
            f.write(struct.pack("<i", t) + np.asarray(pose, np.float32).tobytes() + g.tobytes() + d.tobytes())
    args = [exe, str(W), str(H)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]
    r = subprocess.run(args + [fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.frombuffer(open(fout, "rb").read(), np.uint8)
    pitch = 3 * W + 5
    assert len(raw) == len(fr) * H * pitch + H * 3 * W
    pattern = (np.arange(H * pitch, dtype=np.int64) * 7 ^ 0xA5).astype(np.uint8).reshape(H, pitch)
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=200000)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    for t, (pose, g, d) in enumerate(fr):
        ctx.fuse_frame_resident(t, g, d, pose)
        want = check_image(ctx, 0, t % 2, g, d, f"C++ stream frame {t}")
        got = raw[t * H * pitch:(t + 1) * H * pitch].reshape(H, pitch)
        assert got[:, :3 * W].tobytes() == want.tobytes(), f"ResidentSurfelPool::superpixel_image frame {t}"
        assert got[:, 3 * W:].tobytes() == pattern[:, 3 * W:].tobytes(), "padding bytes written"
    ctx.close()
    # dsm::FusionFunctions::superpixel_image after fuse_initialize_map of the last frame: superpixels depend on the
    # image alone, so it is the resident stream's last image
    assert raw[len(fr) * H * pitch:].tobytes() == want.tobytes()
