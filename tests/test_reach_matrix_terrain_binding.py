"""capi.Context.reach_matrix_enqueue_terrain hands the library the points as n x 3 contiguous float64, their count, the
radius and the approach exactly as reach_matrix_enqueue does, and reach_matrix_wait reads back the sites and the matrix
of whichever kind of job ran last, as terrain and field jobs alternate."""
import ctypes
import types

import numpy as np

import pyoracle_reach_matrix as RM
from densesurfelmapping_b200 import capi


def test_arguments_and_results_as_terrain_and_field_jobs_alternate():
    calls, bufs = [], {}

    def enqueue(kind):
        def call(h, points, n, radius, approach):
            p = np.ctypeslib.as_array(ctypes.cast(points, ctypes.POINTER(ctypes.c_double)), (n, 3)).copy() if points else None
            calls.append((kind, h, p, n, radius, approach))
            bufs["sites"] = np.zeros(n, capi.REACH_SITE_DTYPE)
            bufs["sites"]["voxel"] = np.arange(n) * (3 if kind == "terrain" else 5)
            bufs["matrix"] = (np.arange(n * n, dtype=np.uint32) + (7 if kind == "terrain" else 11)).reshape(n, n)
            return 0
        return call

    def wait(h, info, ps, pm):
        rec = np.zeros(1, capi.REACH_MATRIX_INFO_DTYPE)
        rec["n_sites"] = len(bufs["sites"])
        ctypes.memmove(info, rec.ctypes.data, rec.itemsize)
        ps._obj.value, pm._obj.value = bufs["sites"].ctypes.data, bufs["matrix"].ctypes.data
        return 0

    lib = types.SimpleNamespace(dsm_reach_matrix_enqueue=enqueue("field"), dsm_reach_matrix_enqueue_terrain=enqueue("terrain"),
                                dsm_reach_matrix_wait=wait)
    ctx = capi.Context.__new__(capi.Context)
    ctx.h, ctx.lib = 1234, lib
    rng = np.random.default_rng(0)
    for k, kind in enumerate(("terrain", "field", "terrain", "terrain", "field")):
        want_pts = rng.normal(size=(k + 2, 3))
        given = want_pts.tolist() if k == 2 else np.asfortranarray(want_pts)   # any array-like of points
        if kind == "terrain":
            ctx.reach_matrix_enqueue_terrain(given, np.float32(0.25), np.int64(3))
        else:
            ctx.reach_matrix_enqueue(given, 0.25, 3)
        got_kind, h, p, n, radius, approach = calls[-1]
        assert (got_kind, h, n, approach) == (kind, 1234, len(want_pts), 3)
        assert type(radius) is float and radius == 0.25 and type(approach) is int
        assert p.tobytes() == want_pts.tobytes()
        info, sites, M = ctx.reach_matrix_wait()
        assert info["n_sites"] == n and sites.dtype == capi.REACH_SITE_DTYPE and M.dtype == np.uint32 and M.shape == (n, n)
        assert sites.tobytes() == bufs["sites"].tobytes() and M.tobytes() == bufs["matrix"].tobytes()
        assert not np.shares_memory(M, bufs["matrix"]) and not np.shares_memory(sites, bufs["sites"])
    assert capi.REACH_SITE_DTYPE == RM.SITE_DTYPE and capi.REACH_MATRIX_INFO_DTYPE == RM.MATRIX_INFO_DTYPE
