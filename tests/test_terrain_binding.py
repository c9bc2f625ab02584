"""capi.Context.terrain_wait hands out the four planes of the terrain grid [m2][m1][m0] with their dtypes, read from the
library's pinned buffers in the order of include/dsm.h, and its header record is the model's."""
import ctypes
import types

import numpy as np

import pyoracle_terrain as TR
from densesurfelmapping_b200 import capi


def test_planes_come_back_in_the_terrain_grid_shape_with_their_dtypes():
    m = (5, 1, 3)    # up along y
    cells = 15
    bufs = [np.arange(cells, dtype=np.int16) - 1, (np.arange(cells) % 3).astype(np.uint8), np.arange(cells, dtype=np.uint8) * 2,
            np.linspace(0.0, 1.4, cells, dtype=np.float32)]

    def wait(h, info, *ptrs):
        rec = np.zeros(1, capi.TERRAIN_INFO_DTYPE)
        rec["m"], rec["up"], rec["headroom"] = m, -2, 3
        ctypes.memmove(info, rec.ctypes.data, rec.itemsize)
        for p, b in zip(ptrs, bufs):
            p._obj.value = b.ctypes.data
        return 0

    stub = types.SimpleNamespace(h=None, lib=types.SimpleNamespace(dsm_terrain_wait=wait), _waited=lambda rc, name, f: f())
    info, level, status, step, clearance = capi.Context.terrain_wait(stub)
    assert info["up"] == -2 and info["headroom"] == 3 and list(info["m"]) == list(m)
    for got, want in zip((level, status, step, clearance), bufs):
        assert got.shape == (3, 1, 5) and got.dtype == want.dtype
        assert got.reshape(-1).tobytes() == want.tobytes()
        assert not np.shares_memory(got, want)   # copies of the pinned buffers
    assert capi.TERRAIN_INFO_DTYPE == TR.INFO_DTYPE and TR.INFO_DTYPE.itemsize == 64
