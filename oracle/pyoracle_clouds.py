"""TEST INFRASTRUCTURE ONLY -- the node's raw and neighbourhood cloud publishers, for tests/test_node_clouds.py and
tests/test_gpu_node_clouds.py.

  raw_cloud       publish_raw_pointcloud (surfel_map.cpp:1115-1151) restated in numpy float32, operation by operation
  RefMapClouds    pyoracle.RefMap over oracle/_ref/libdsm_refmap_clouds.so (oracle/clouds.mk, ref_map_clouds.cpp): the
                  reference's SurfelMap with two more hooks, publish_raw() and driftfree_poses()
"""
import ctypes
import os
import subprocess

import numpy as np

import pyoracle

LIBNAME = "libdsm_refmap_clouds.so"


def build(verbose=False):
    """Build libdsm_refmap_clouds.so where the reference sources exist (see oracle/clouds.mk)."""
    r = subprocess.run(["make", "-C", pyoracle.HERE, "-f", "clouds.mk", "clouds"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed (clouds.mk)")


def have_refmap_clouds():
    return os.path.exists(os.path.join(pyoracle.REFDIR, LIBNAME))


def raw_rotation(pose7):
    """R = Quaternionf((float)qw, (float)qx, (float)qy, (float)qz).toRotationMatrix() (not normalised; Eigen's formula,
    oracle/shim/Eigen/Eigen:266-277) and T = (float)position, as publish_raw_pointcloud forms them (:1117-1127)."""
    f = np.float32
    p = np.asarray(pose7, np.float64).reshape(7)
    qx, qy, qz, qw = (f(v) for v in p[3:7])
    tx, ty, tz = f(2) * qx, f(2) * qy, f(2) * qz
    twx, twy, twz = tx * qw, ty * qw, tz * qw
    txx, txy, txz = tx * qx, ty * qx, tz * qx
    tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
    R = [[f(1) - (tyy + tzz), txy - twz, txz + twy],
         [txy + twz, f(1) - (txx + tzz), tyz - twx],
         [txz - twy, tyz + twx, f(1) - (txx + tyy)]]
    return R, p[:3].astype(f)


def raw_cloud(cam, gray, depth, pose7):
    """publish_raw_pointcloud (surfel_map.cpp:1115-1151): [W*H, 4] float32 x, y, z, intensity.  Column i is the outer
    loop, row j the inner one (point i*H + j); every pixel is emitted, a hole (depth 0) lands on T."""
    f = np.float32
    R, T = raw_rotation(pose7)
    d = np.ascontiguousarray(np.asarray(depth, f).T)                # [W][H]: the loop order
    i = np.arange(cam.width, dtype=f)[:, None]
    j = np.arange(cam.height, dtype=f)[None, :]
    c0 = (i - f(cam.cx)) * d / f(cam.fx)                              # (i - cam_cx) * depth_value / cam_fx   :1135
    c1 = (j - f(cam.cy)) * d / f(cam.fy)                              # :1136
    out = np.empty((cam.width, cam.height, 4), f)
    for r in range(3):                                               # rotation_R * cam_point + translation_T :1139
        out[..., r] = ((R[r][0] * c0 + R[r][1] * c1) + R[r][2] * d) + T[r]
    out[..., 3] = np.asarray(gray, np.uint8).T                       # reference.at<uchar>(j, i)  :1145
    return out.reshape(-1, 4)


class RefMapClouds(pyoracle.RefMap):
    """pyoracle.RefMap (the reference's SurfelMap, its own CPU FusionFunctions) loaded from libdsm_refmap_clouds.so,
    which adds publish_raw() and driftfree_poses()."""

    def __init__(self, cam, drift_free_poses=10):
        path = os.path.join(pyoracle.REFDIR, LIBNAME)
        if not os.path.exists(path):
            build()
        lib = ctypes.CDLL(path)
        # RefMap.__init__ resolves its library through pyoracle._lib: hand it this one
        load = pyoracle._lib
        pyoracle._lib = lambda name: lib
        try:
            super().__init__(cam, drift_free_poses)
        finally:
            pyoracle._lib = load
        vp, ci = ctypes.c_void_p, ctypes.c_int
        lib.dsmmap_publish_raw.argtypes = [vp, vp, vp, vp]
        lib.dsmmap_driftfree_poses.argtypes = [vp, ci, ci, vp, ci]
        lib.dsmmap_driftfree_poses.restype = ci

    def publish_raw(self, gray, depth, pose7):
        """publish_raw_pointcloud(depth, gray, pose); returns what it published on ~raw_pointcloud, [W*H, 4] float32."""
        gray = np.ascontiguousarray(gray, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        p = np.ascontiguousarray(pose7, np.float64).reshape(7)
        self.lib.dsmmap_publish_raw(self.h, gray.ctypes.data, depth.ctypes.data, p.ctypes.data)
        return self.published("raw_pointcloud", cap=self.cam.width * self.cam.height)

    def driftfree_poses(self, root, driftfree_range):
        """get_driftfree_poses(root, list, range) (surfel_map.cpp:1643-1680): the BFS list, in BFS order."""
        out = np.zeros(max(self.num_poses(), 1), np.int32)
        n = self.lib.dsmmap_driftfree_poses(self.h, int(root), int(driftfree_range), out.ctypes.data, len(out))
        assert n <= len(out)
        return out[:n].tolist()
