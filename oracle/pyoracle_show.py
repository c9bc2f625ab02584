"""TEST INFRASTRUCTURE ONLY -- FusionFunctions::debug_show (fusion_functions.cpp:977-1006), the superpixel normal image,
for tests/test_superpixel_image.py and tests/test_gpu_superpixel_image.py.

  superpixel_image  debug_show restated in numpy: the exact double product and the reference build's uchar conversion
  RefShow           the serial reference (pyoracle.RefSerial) loaded from oracle/_ref/libdsm_ref_show.so (oracle/show.mk,
                    ref_debug_show.cpp), which adds debug_show(): the image the reference hands to cv::imshow
"""
import ctypes
import os
import subprocess

import numpy as np

import pyoracle
from densesurfelmapping_b200.elements import SEED_DTYPE

LIBNAME = "libdsm_ref_show.so"


def build(verbose=False):
    """Build libdsm_ref_show.so where the reference sources exist (see oracle/show.mk)."""
    r = subprocess.run(["make", "-C", pyoracle.HERE, "-f", "show.mk", "show"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed (show.mk)")


def have_ref_show():
    return os.path.exists(os.path.join(pyoracle.REFDIR, LIBNAME))


def channel(n):
    """`uchar = fabs(n) * 255` (:986-988) as the reference's x86-64 build computes it (cvtss2sd, mulsd, cvttsd2si into a
    32-bit register, low byte stored): the product of the float promoted to double is exact; the truncation to int32
    gives INT_MIN for NaN and for anything >= 2^31, whose low byte is 0."""
    v = np.abs(np.asarray(n, np.float32).astype(np.float64)) * 255.0
    ok = v < 2.0 ** 31                                               # False for NaN
    t = np.trunc(np.where(ok, v, 0.0)).astype(np.int64)
    return np.where(ok, t & 0xFF, 0).astype(np.uint8)


def superpixel_image(labels, seeds):
    """debug_show over labels [H][W] (superpixel_index) and seeds (Superpixel_seed records): [H][W][3] uint8,
    {|norm_x|, |norm_y|, |norm_z|} * 255 of the pixel's seed, black where the right or the lower neighbour's label
    differs (:991-1000)."""
    lab = np.asarray(labels, np.int32)
    seeds = np.asarray(seeds, SEED_DTYPE)
    colour = np.stack([channel(seeds["norm_x"]), channel(seeds["norm_y"]), channel(seeds["norm_z"])], axis=1)
    img = colour[lab]
    edge = np.zeros(lab.shape, bool)
    edge[:, :-1] |= lab[:, 1:] != lab[:, :-1]
    edge[:-1, :] |= lab[1:, :] != lab[:-1, :]
    img[edge] = 0
    return img


class RefShow(pyoracle._Base):
    """The serial reference with a debug_show hook: superpixels() / fuse() as pyoracle.RefSerial, then debug_show()."""
    prefix = "dsmref_"
    libname = LIBNAME

    def __init__(self, cam):
        if not have_ref_show():
            build()
        super().__init__(cam)
        self.lib.dsmref_debug_show.argtypes = [ctypes.c_void_p] * 4
        self.lib.dsmref_debug_show.restype = ctypes.c_int

    def debug_show(self, labels=None, seeds=None):
        """debug_show() on the context's labels and seeds, or on the given ones (which then replace them); returns the
        [H][W][3] uint8 image it showed."""
        H, W = self.cam.height, self.cam.width
        if labels is not None:
            labels = np.ascontiguousarray(labels, np.int32)
            assert labels.shape == (H, W)
        if seeds is not None:
            seeds = np.ascontiguousarray(seeds, SEED_DTYPE)
            assert seeds.shape == (self.S,)
        out = np.zeros((H, W, 3), np.uint8)
        rc = self.lib.dsmref_debug_show(self.h, None if labels is None else labels.ctypes.data,
                                        None if seeds is None else seeds.ctypes.data, out.ctypes.data)
        assert rc == 0, "debug_show showed no H x W x 3 image"
        return out
