"""capi.Context.reach_wait hands out the cost grid in the shape of the grid the last enqueued job ran on: [m2][m1][m0] of
the terrain grid after reach_enqueue_terrain and [nz][ny][nx] after reach_enqueue, as the two kinds alternate, with the
same record dtypes either way."""
import ctypes
import types

import numpy as np
import pytest

import pyoracle_reach as R
from densesurfelmapping_b200 import capi


@pytest.mark.parametrize("up", (1, -1, 2, -2, 3, -3))
def test_cost_shapes_follow_the_kind_of_job_as_terrain_and_field_jobs_alternate(up):
    nx, ny, nz = 5, 4, 3
    m = [nx, ny, nz]
    m[abs(up) - 1] = 1
    cells = m[0] * m[1] * m[2]
    bufs = {}

    def enqueue(kind):
        def call(h, start, radius, approach, goals, n_goals, with_frontiers, host_copy):
            n = cells if kind == "terrain" else nx * ny * nz
            bufs["cost"] = np.arange(n, dtype=np.uint32) * 7
            bufs["rec"] = np.zeros(2, capi.REACH_TARGET_DTYPE)
            bufs["rec"]["target"] = (3, n - 1)
            bufs["path"] = np.arange(4, dtype=np.int32)
            return 0
        return call

    def wait(h, info, pt, pp, pc):
        rec = np.zeros(1, capi.REACH_INFO_DTYPE)
        rec["n_targets"], rec["n_path_voxels"] = 2, 4
        ctypes.memmove(info, rec.ctypes.data, rec.itemsize)
        pt._obj.value, pp._obj.value, pc._obj.value = bufs["rec"].ctypes.data, bufs["path"].ctypes.data, bufs["cost"].ctypes.data
        return 0

    lib = types.SimpleNamespace(dsm_reach_enqueue=enqueue("field"), dsm_reach_enqueue_terrain=enqueue("terrain"), dsm_reach_wait=wait,
                                dsm_terrain_enable=lambda h, up: 0)
    ctx = capi.Context.__new__(capi.Context)
    ctx.h, ctx.lib, ctx._field_shape = None, lib, (nz, ny, nx)
    ctx.terrain_enable(up)
    for kind in ("terrain", "field", "terrain", "terrain", "field"):
        if kind == "terrain":
            ctx.reach_enqueue_terrain((0.0, 0.0, 0.0), 0.0, 0, [(1.0, 2.0, 3.0)], host_copy=True)
        else:
            ctx.reach_enqueue((0.0, 0.0, 0.0), 0.0, 0, None, host_copy=True)
        info, targets, path, cost = ctx.reach_wait()
        want = (m[2], m[1], m[0]) if kind == "terrain" else (nz, ny, nx)
        assert cost.shape == want and cost.dtype == np.uint32, kind
        assert cost.reshape(-1).tobytes() == bufs["cost"].tobytes() and not np.shares_memory(cost, bufs["cost"])
        assert targets.dtype == capi.REACH_TARGET_DTYPE and list(targets["target"]) == [3, cost.size - 1]
        assert path.dtype == np.int32 and len(path) == 4 and info.dtype == capi.REACH_INFO_DTYPE
    assert capi.REACH_TARGET_DTYPE == R.TARGET_DTYPE and capi.REACH_INFO_DTYPE == R.INFO_DTYPE
