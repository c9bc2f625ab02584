"""TEST INFRASTRUCTURE ONLY -- the node's per-frame window step (SurfelMap::move_add_surfels, surfel_map.cpp:1458-1595),
for tests/test_window_step.py and tests/test_gpu_window_stream.py.

  WindowModel     the window step restated in numpy on the three things the device keeps: the pool (local_surfels), the
                  inactive store (every pose's attached_surfels, dense in retirement order) and its segment list
  RefMapWindow    pyoracle.RefMap over oracle/_ref/libdsm_refmap_window[_b200].so (oracle/window.mk, ref_map_window.cpp):
                  the reference's SurfelMap with three more hooks, window_lists(), pending_frame() and images()
"""
import ctypes
import os
import subprocess

import numpy as np

import pyoracle
from pyoracle import SURFEL_DTYPE


def build(verbose=False):
    """Build libdsm_refmap_window[_b200].so where the reference sources exist (see oracle/window.mk)."""
    r = subprocess.run(["make", "-C", pyoracle.HERE, "-f", "window.mk", "window"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed (window.mk)")


def libname(b200=False):
    return "libdsm_refmap_window_b200.so" if b200 else "libdsm_refmap_window.so"


def have_refmap_window(b200=False):
    return os.path.exists(os.path.join(pyoracle.REFDIR, libname(b200)))


def cloud(surfels):
    """inactive_pointcloud's points of these surfels: {px, py, pz, color} (surfel_map.cpp:1485-1490)."""
    s = np.asarray(surfels, SURFEL_DTYPE)
    return np.stack([s["px"], s["py"], s["pz"], s["color"]], axis=1).astype(np.float32).reshape(-1, 4)


class WindowModel:
    """move_add_surfels on (pool, store, segments).  retire: the live surfels of each keyframe, in list order, pool order
    within a keyframe, become one segment at the end of the store (none for a keyframe without any) and are flagged
    dead in the pool.  reactivate: each keyframe's segments, in list order, go back to the end of the pool and leave
    the store, which closes up in order."""

    def __init__(self, pool=None):
        self.pool = np.zeros(0, SURFEL_DTYPE) if pool is None else np.array(pool, SURFEL_DTYPE)
        self.store = np.zeros(0, SURFEL_DTYPE)
        self.segs = []  # (keyframe, offset, count), retirement order

    def step(self, retire, reactivate):
        for kf in retire:
            sel = (self.pool["update_times"] > 0) & (self.pool["last_update"] == kf)
            out = self.pool[sel].copy()
            self.pool["update_times"][sel] = 0
            if len(out):
                self.segs.append((int(kf), len(self.store), len(out)))
                self.store = np.concatenate([self.store, out])
        back = []
        for kf in reactivate:
            keep, parts, ofs = [], [], 0
            for k, o, c in self.segs:
                if k == kf:
                    back.append(self.store[o:o + c])
                else:
                    parts.append(self.store[o:o + c])
                    keep.append((k, ofs, c))
                    ofs += c
            self.segs = keep
            self.store = np.concatenate(parts) if parts else np.zeros(0, SURFEL_DTYPE)
        if back:
            self.pool = np.concatenate([self.pool] + back)

    def attached(self, kf):
        parts = [self.store[o:o + c] for k, o, c in self.segs if k == kf]
        return np.concatenate(parts) if parts else np.zeros(0, SURFEL_DTYPE)


class RefMapWindow(pyoracle.RefMap):
    """pyoracle.RefMap loaded from libdsm_refmap_window[_b200].so, which adds window_lists(), pending_frame() and
    images().  b200=True: the node over the product adapter (needs a GPU)."""

    def __init__(self, cam, drift_free_poses=10, b200=False):
        path = os.path.join(pyoracle.REFDIR, libname(b200))
        if not os.path.exists(path):
            build()
        lib = ctypes.CDLL(path)
        load = pyoracle._lib
        pyoracle._lib = lambda name: lib  # RefMap.__init__ resolves its library through pyoracle._lib
        try:
            super().__init__(cam, drift_free_poses)
        finally:
            pyoracle._lib = load
        vp, ci = ctypes.c_void_p, ctypes.c_int
        lib.dsmmap_window_lists.argtypes = [vp, ci, vp, vp, vp, vp, ci]
        lib.dsmmap_window_lists.restype = None
        lib.dsmmap_pending_frame.argtypes = [vp, vp, vp, vp, vp, vp, ci]
        lib.dsmmap_pending_frame.restype = ci
        lib.dsmmap_images.argtypes = [vp, ctypes.c_double, vp, vp]
        lib.dsmmap_images.restype = None

    def images(self, stamp, gray, depth):
        """The image and depth callbacks of a frame whose pose was fed with gray=None: the node runs move_add_surfels
        and fuse_map for it."""
        gray = np.ascontiguousarray(gray, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        self.lib.dsmmap_images(self.h, float(stamp), gray.ctypes.data, depth.ctypes.data)

    def window_lists(self, root):
        """get_add_remove_poses(root): (poses_to_remove, poses_to_add) as move_add_surfels(root) would use them."""
        cap = max(self.num_poses(), 1)
        add, rem = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        na, nr = ctypes.c_int(0), ctypes.c_int(0)
        self.lib.dsmmap_window_lists(self.h, int(root), add.ctypes.data, ctypes.byref(na), rem.ctypes.data, ctypes.byref(nr), cap)
        return rem[:nr.value].tolist(), add[:na.value].tolist()

    def pending_frame(self):
        """For the frame whose pose has arrived and whose images have not: (reference index, fuse pose as the
        column-major float32[16] fuse_map receives, poses_to_remove, poses_to_add), or None."""
        cap = max(self.num_poses(), 1)
        pose = np.zeros(16, np.float32)
        add, rem = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        na, nr = ctypes.c_int(0), ctypes.c_int(0)
        ref = self.lib.dsmmap_pending_frame(self.h, pose.ctypes.data, add.ctypes.data, ctypes.byref(na), rem.ctypes.data,
                                            ctypes.byref(nr), cap)
        if ref < 0:
            return None
        return ref, pose, rem[:nr.value].tolist(), add[:na.value].tolist()
