"""capi.Context.viewpoint_enqueue_terrain hands the library the camera, the rotations as n x 9 contiguous float64, the
clusters as int32, the parameters and eye exactly as viewpoint_enqueue hands its arguments (eye last), and viewpoint_wait
reads back the header, records and slots of whichever kind of job ran last, as terrain and field jobs alternate."""
import ctypes
import types

import numpy as np

import pyoracle_viewpoint as V
from densesurfelmapping_b200 import capi


def test_arguments_and_results_as_terrain_and_field_jobs_alternate():
    calls, bufs = [], {}

    def enqueue(kind):
        def call(h, cam, rot, n_rot, cl, n_cl, prm, *eye):
            c, p = cam._obj, prm._obj
            R = np.ctypeslib.as_array(ctypes.cast(rot, ctypes.POINTER(ctypes.c_double)), (n_rot, 9)).copy()
            C = np.ctypeslib.as_array(ctypes.cast(cl, ctypes.POINTER(ctypes.c_int32)), (n_cl,)).copy() if cl else np.zeros(0, np.int32)
            calls.append((kind, h, (c.fx, c.fy, c.cx, c.cy, c.width, c.height, c.max_range, c.unknown_blocks), R, C,
                          tuple(getattr(p, f) for f, _ in capi.DsmViewpointParams._fields_), eye))
            top_k = p.top_k
            bufs["recs"] = np.zeros(n_cl, capi.VIEWPOINT_CLUSTER_DTYPE)
            bufs["recs"]["cluster"] = C
            bufs["slots"] = np.zeros(n_cl * top_k, capi.VIEWPOINT_DTYPE)
            bufs["slots"]["voxel"] = np.arange(n_cl * top_k) * (3 if kind == "terrain" else 5)
            bufs["info"] = np.zeros(1, capi.VIEWPOINT_INFO_DTYPE)
            bufs["info"]["n_clusters"], bufs["info"]["top_k"] = n_cl, top_k
            return 0
        return call

    def wait(h, info, pc, pv):
        ctypes.memmove(info, bufs["info"].ctypes.data, bufs["info"].itemsize)
        pc._obj.value, pv._obj.value = bufs["recs"].ctypes.data, bufs["slots"].ctypes.data
        return 0

    lib = types.SimpleNamespace(dsm_viewpoint_enqueue=enqueue("field"), dsm_viewpoint_enqueue_terrain=enqueue("terrain"),
                                dsm_viewpoint_wait=wait)
    ctx = capi.Context.__new__(capi.Context)
    ctx.h, ctx.lib = 1234, lib
    rng = np.random.default_rng(0)
    cam = (2.0, 3.0, 1.5, 1.0, 4, 3, np.float32(1.25), 1)
    for k, kind in enumerate(("terrain", "field", "terrain", "terrain", "field")):
        rot = rng.normal(size=(k + 1, 9))
        cl = np.arange(k + 2, dtype=np.int64)[::-1]
        prm = (1, 4, 0, 2, 64, 1, k + 1, k % 2, np.float64(0.3))
        given = rot.tolist() if k == 2 else np.asfortranarray(rot)
        if kind == "terrain":
            ctx.viewpoint_enqueue_terrain(cam, given, cl.tolist(), prm, np.int64(k + 1))
        else:
            ctx.viewpoint_enqueue(cam, given, cl, prm)
        got_kind, h, c, R, C, p, eye = calls[-1]
        assert (got_kind, h) == (kind, 1234)
        assert c == (2.0, 3.0, 1.5, 1.0, 4, 3, 1.25, 1)
        assert R.tobytes() == rot.tobytes() and C.tolist() == cl.tolist()
        assert p[:8] == prm[:8] and abs(p[8] - 0.3) < 1e-7 and p[9] == 0
        assert eye == ((k + 1,) if kind == "terrain" else ()) and all(type(e) is int for e in eye)
        info, recs, slots = ctx.viewpoint_wait()
        assert info["n_clusters"] == len(cl) and slots.shape == (len(cl), k + 1)
        assert recs.tobytes() == bufs["recs"].tobytes() and slots.tobytes() == bufs["slots"].tobytes()
        assert not np.shares_memory(slots, bufs["slots"])
    assert capi.VIEWPOINT_DTYPE == V.VIEWPOINT_DTYPE and capi.VIEWPOINT_INFO_DTYPE == V.INFO_DTYPE
