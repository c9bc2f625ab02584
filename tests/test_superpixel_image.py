"""The superpixel normal image of FusionFunctions::debug_show (fusion_functions.cpp:977-1006), CPU side.

debug_show is restated in numpy (oracle/pyoracle_show.py::superpixel_image).  The restatement is pinned by CRC32s of the
image the reference's own debug_show draws (tests/golden/superpixel_image_checksums.json, minted by
tests/golden/make_golden_superpixel_image.py) and, where the reference is built, compared with it byte for byte: on the
labels and seeds of real frames, and on injected seeds whose normals sit on and next to the conversion's integer steps.
The device side is tests/test_gpu_superpixel_image.py."""
import json
import os

import numpy as np
import pytest

import pyoracle
import pyoracle_show
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SEED_DTYPE, num_seeds
from node_drive import build_adapter
from util import CAM, GOLD, crc

needs_ref_show = pytest.mark.skipif(not pyoracle_show.have_ref_show(),
                                    reason="oracle/_ref/libdsm_ref_show.so not built (needs the reference sources)")

CASES = ["vga", "kitti", "vga_flat"]


def image_cases():
    """name -> (camera, gray, depth): VGA and KITTI 1226x370 synthetic frames, and a flat VGA frame whose superpixels
    include NaN normals (all pixel normals zero, DESIGN.md 1.3) and rejected plane fits (zero normals)."""
    def frame(cam, t, flat=False):
        return synth.make_frame(cam, t, synth.pose_stream(t), flat=flat)
    return {"vga": (synth.VGA,) + frame(synth.VGA, 3),
            "kitti": (synth.KITTI,) + frame(synth.KITTI, 5),
            "vga_flat": (synth.VGA,) + frame(synth.VGA, 1, flat=True)}


def golden():
    return json.load(open(os.path.join(GOLD, "superpixel_image_checksums.json")))


def normals(seeds):
    return np.stack([seeds["norm_x"], seeds["norm_y"], seeds["norm_z"]], axis=1)


@pytest.mark.parametrize("case", CASES)
def test_restatement_is_pinned(case):
    cam, gray, depth = image_cases()[case]
    orc = pyoracle.Restatement(cam)          # labels and seeds byte-identical to the serial reference (test_oracle.py)
    labels, seeds = orc.superpixels(gray, depth)
    orc.close()
    img = pyoracle_show.superpixel_image(labels, seeds)
    assert img.shape == (cam.height, cam.width, 3) and img.dtype == np.uint8
    n = normals(seeds)
    if case == "vga_flat":
        assert np.isnan(n).any(1).sum() > 0 and (n == 0).all(1).sum() > 0
    # spot checks of the two rules: an interior pixel of a seed takes its colour, a pixel left of a boundary is black
    y, x = 4 + 8 * 7, 4 + 8 * 9
    s = labels[y, x]
    if labels[y, x + 1] == s and labels[y + 1, x] == s and not np.isnan(n[s]).any():
        assert (img[y, x] == np.floor(np.abs(n[s].astype(np.float64)) * 255)).all()
    ys, xs = np.nonzero(labels[:, :-1] != labels[:, 1:])
    assert (img[ys, xs] == 0).all()
    assert crc(img.tobytes()) == golden()[case]


@needs_ref_show
@pytest.mark.parametrize("case", CASES)
def test_restatement_equals_reference_debug_show(case):
    cam, gray, depth = image_cases()[case]
    m = pyoracle_show.RefShow(cam)
    labels, seeds = m.superpixels(gray, depth)
    want = m.debug_show()
    assert want.tobytes() == pyoracle_show.superpixel_image(labels, seeds).tobytes()
    # fed back the same arrays, the hook draws the same image
    assert m.debug_show(labels, seeds).tobytes() == want.tobytes()
    m.close()


def adversarial_normals():
    """Components on and one ulp either side of k/255 (where the truncation steps), the ends of the range, signed
    zeros, negatives, NaN, inf, and values whose product leaves uchar (> 1) or int32 (>= 2^31 / 255)."""
    f = np.float32
    vals = []
    for k in (0, 1, 2, 3, 17, 51, 100, 127, 128, 129, 200, 254, 255):
        v = f(k) / f(255)
        vals += [v, np.nextafter(v, f(2)), np.nextafter(v, f(-2)), -v]
    vals += [f(1), np.nextafter(f(1), f(2)), f(-1), f(0), f(-0.0), f(np.nan), -f(np.nan), f(np.inf), -f(np.inf),
             f(1.5), f(2), f(-3.25), f(8421504.5), f(3e7), f(1e-30), f(np.finfo(np.float32).tiny / 4)]
    return np.array(vals, np.float32)


def adversarial_seeds(S, rng):
    seeds = np.zeros(S, SEED_DTYPE)
    v = adversarial_normals()
    for f in ("norm_x", "norm_y", "norm_z"):
        seeds[f] = v[rng.integers(0, len(v), S)]
    seeds["x"], seeds["y"] = rng.uniform(0, 100, S), rng.uniform(0, 100, S)
    seeds["mean_depth"] = rng.uniform(0.5, 10, S)
    return seeds


def adversarial_labels(cam, S, rng):
    """Blocks of random seeds with jagged edges, and boundaries on the last row and the last column."""
    H, W = cam.height, cam.width
    lab = rng.integers(0, S, (H // 5 + 1, W // 7 + 1)).repeat(5, 0).repeat(7, 1)[:H, :W].astype(np.int32)
    lab[rng.random((H, W)) < 0.02] = rng.integers(0, S)
    lab[H - 1, ::3] = (lab[H - 1, ::3] + 1) % S          # last row differs from its left / right neighbours
    lab[::4, W - 1] = (lab[::4, W - 1] + 2) % S          # last column differs from the row above / below
    lab[H - 1, W - 1] = S - 1
    return lab


def test_restatement_channel_rule():
    v = adversarial_normals()
    got = pyoracle_show.channel(v).astype(np.int64)
    d = np.abs(v.astype(np.float64)) * 255
    for x, g, p in zip(v, got, d):
        if np.isnan(p) or p >= 2 ** 31:
            assert g == 0, x
        else:
            assert g == int(p) % 256, x
    k = np.arange(256)
    assert (pyoracle_show.channel(np.float32(k) / np.float32(255)) <= k).all()


@needs_ref_show
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_equals_reference_on_injected_seeds(seed):
    rng = np.random.default_rng(seed)
    cam = CAM
    S = num_seeds(cam.width, cam.height)
    seeds = adversarial_seeds(S, rng)
    labels = adversarial_labels(cam, S, rng)
    m = pyoracle_show.RefShow(cam)
    want = m.debug_show(labels, seeds)
    m.close()
    got = pyoracle_show.superpixel_image(labels, seeds)
    assert got.tobytes() == want.tobytes(), f"{(got != want).any(2).sum()} pixels differ"
    # the injected values reach the picture: NaN and large components give 0, 2.0 gives 510 & 0xff
    assert (want[-1, :-1] == 0).any() and (want[:-1, -1] == 0).any()


@needs_ref_show
def test_nan_normal_converts_to_zero_in_the_reference():
    """The value the oracle build gives a NaN channel (the contract dsm.h documents): 0, like the restatement."""
    cam = CAM
    S = num_seeds(cam.width, cam.height)
    seeds = np.zeros(S, SEED_DTYPE)
    seeds["norm_x"], seeds["norm_y"], seeds["norm_z"] = np.nan, np.float32(128) / np.float32(255), np.float32(2)
    labels = np.zeros((cam.height, cam.width), np.int32)
    m = pyoracle_show.RefShow(cam)
    img = m.debug_show(labels, seeds)
    m.close()
    assert (img[..., 0] == 0).all() and (img[..., 1] == 128).all() and (img[..., 2] == 254).all()


def test_superpixel_image_helper_compiles_and_fails_loudly_without_gpu(tmp_path):
    import subprocess
    import torch
    exe = build_adapter("superpixel_image_main")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_gpu_superpixel_image.py")
    cam = CAM
    args = [exe, str(cam.width), str(cam.height)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]
    r = subprocess.run(args + [str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "no usable CUDA device" in r.stderr
