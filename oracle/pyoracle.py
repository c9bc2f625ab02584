"""TEST INFRASTRUCTURE ONLY — ctypes access to the CPU oracles.

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs.  Never from the product path (the product is the CUDA library
behind include/dsm.h and fails loudly if it is missing).

Three libraries under oracle/_ref/ (built by oracle/Makefile):
  libdsm_ref_serial.so  the reference's own fusion_functions.cpp, thread bodies inline  -> PARITY ORACLE
  libdsm_ref_mt.so      the reference's own fusion_functions.cpp as shipped (10 threads) -> timed CPU baseline
  libdsm_oracle.so      this repo's plain-C restatement (oracle/dsm_oracle.c), pinned to ref_serial
"""
import ctypes
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(HERE, "_ref")

import sys
sys.path.insert(0, os.path.dirname(HERE))
from densesurfelmapping_b200.elements import SEED_DTYPE, SURFEL_DTYPE, num_seeds  # noqa: E402


def build(force=False, verbose=False):
    """Build every oracle library that is out of date, or all of them with force=True: the restatement always, the
    reference variants when the reference sources exist (see oracle/Makefile)."""
    r = subprocess.run(["make", "-C", HERE, "all"] + (["-B"] if force else []), capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed")


def have(libname):
    """Whether oracle/_ref/<libname> is built."""
    return os.path.exists(os.path.join(REFDIR, libname))


def _lib(name):
    path = os.path.join(REFDIR, name)
    if not have(name):
        build()
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    return ctypes.CDLL(path)


_u8p = ctypes.POINTER(ctypes.c_uint8)
_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int32)


class _Base:
    """Common wrapper; both the reference driver and the restatement export the same entry points
    with prefix dsmref_ / dsmor_."""
    prefix = None
    libname = None

    def __init__(self, cam):
        self.cam = cam
        self.lib = _lib(self.libname)
        p = self.prefix
        L = self.lib
        getattr(L, p + "create").restype = ctypes.c_void_p
        getattr(L, p + "create").argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_float] * 6
        getattr(L, p + "destroy").argtypes = [ctypes.c_void_p]
        getattr(L, p + "fuse").restype = ctypes.c_int
        getattr(L, p + "fuse").argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        getattr(L, p + "superpixels").argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        getattr(L, p + "get_labels").argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        getattr(L, p + "get_seeds").argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        getattr(L, p + "get_norm_map").argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        self.h = getattr(L, p + "create")(cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)
        self.S = num_seeds(cam.width, cam.height)

    def close(self):
        if self.h:
            getattr(self.lib, self.prefix + "destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def fuse(self, ref_idx, gray, depth, pose, local):
        """fuse_initialize_map semantics: returns (local_updated, new_surfels)."""
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        pose = np.ascontiguousarray(pose, dtype=np.float32).reshape(16)
        local = np.array(local, dtype=SURFEL_DTYPE, copy=True)
        new = np.zeros(self.S, dtype=SURFEL_DTYPE)
        n = getattr(self.lib, self.prefix + "fuse")(
            self.h, int(ref_idx), gray.ctypes.data, depth.ctypes.data, pose.ctypes.data,
            local.ctypes.data if len(local) else None, len(local), new.ctypes.data, self.S)
        return local, new[:n].copy()

    def superpixels(self, gray, depth):
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        getattr(self.lib, self.prefix + "superpixels")(self.h, gray.ctypes.data, depth.ctypes.data)
        return self.labels(), self.seeds()

    def labels(self):
        out = np.empty((self.cam.height, self.cam.width), dtype=np.int32)
        getattr(self.lib, self.prefix + "get_labels")(self.h, out.ctypes.data)
        return out

    def seeds(self):
        out = np.zeros(self.S, dtype=SEED_DTYPE)
        getattr(self.lib, self.prefix + "get_seeds")(self.h, out.ctypes.data)
        return out

    def norm_map(self):
        out = np.empty((self.cam.height, self.cam.width, 3), dtype=np.float32)
        getattr(self.lib, self.prefix + "get_norm_map")(self.h, out.ctypes.data)
        return out


class RefSerial(_Base):
    prefix = "dsmref_"
    libname = "libdsm_ref_serial.so"


class RefSerialRGBD(_Base):
    """The serial reference compiled with its second constant set (fusion_functions.h:17-21; oracle/ref_driver.cpp, DSM_REF_RGBD)."""
    prefix = "dsmref_"
    libname = "libdsm_ref_serial_rgbd.so"


class RefMT(_Base):
    prefix = "dsmref_"
    libname = "libdsm_ref_mt.so"


CONSTANTS_DRIVE = (0.4, 0.5, 4.0, 0.1)    # fusion_functions.h:13-16
CONSTANTS_RGBD = (0.05, 0.08, 1.0, 0.05)  # fusion_functions.h:18-21


class Restatement(_Base):
    prefix = "dsmor_"
    libname = "libdsm_oracle.so"

    def __init__(self, cam, constants=CONSTANTS_DRIVE):
        super().__init__(cam)
        self.constants = tuple(float(c) for c in constants)
        self.lib.dsmor_set_constants.argtypes = [ctypes.c_double] * 4
        self.lib.dsmor_set_constants.restype = None

    def _select(self):
        self.lib.dsmor_set_constants(*self.constants)  # process-wide in the C file: set before every call of this object

    def fuse(self, *a, **k):
        self._select()
        return super().fuse(*a, **k)

    def superpixels(self, *a, **k):
        self._select()
        return super().superpixels(*a, **k)

    def debug_iters(self, gray, depth, iters, last_with_update=True):
        """seed init + `iters` assign passes (last update_seeds optional); returns (labels, seeds)."""
        self._select()
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        self.lib.dsmor_debug_iters.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        self.lib.dsmor_debug_iters(self.h, gray.ctypes.data, depth.ctypes.data, int(iters), int(bool(last_with_update)))
        return self.labels(), self.seeds()


def fuse_map_poststep(local, new):
    """SurfelMap::fuse_map post-step (surfel_map.cpp:1077-1109) via the restatement; returns the new pool."""
    lib = _lib("libdsm_oracle.so")
    lib.dsmor_fuse_map_poststep.restype = ctypes.c_int
    lib.dsmor_fuse_map_poststep.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    buf = np.zeros(len(local) + len(new) + 1, dtype=SURFEL_DTYPE)
    buf[:len(local)] = local
    new = np.ascontiguousarray(new, dtype=SURFEL_DTYPE)
    n = lib.dsmor_fuse_map_poststep(buf.ctypes.data, len(local), new.ctypes.data if len(new) else None, len(new))
    return buf[:n].copy()


def retire(local, kf):
    """move_add_surfels removal half (surfel_map.cpp:1479-1497) via the restatement: returns (local_after, retired)."""
    lib = _lib("libdsm_oracle.so")
    lib.dsmor_retire.restype = ctypes.c_int
    lib.dsmor_retire.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    loc = np.array(local, dtype=SURFEL_DTYPE, copy=True)
    out = np.zeros(len(loc) + 1, dtype=SURFEL_DTYPE)
    n = lib.dsmor_retire(loc.ctypes.data if len(loc) else None, len(loc), int(kf), out.ctypes.data)
    return loc, out[:n].copy()


def warp_active(surfels, W_colmajor):
    """warp_active_surfels_cpu_kernel (surfel_map.cpp:750-789) via the restatement."""
    lib = _lib("libdsm_oracle.so")
    lib.dsmor_warp_active.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    out = np.array(surfels, dtype=SURFEL_DTYPE, copy=True)
    w = np.ascontiguousarray(W_colmajor, dtype=np.float32).reshape(16)
    lib.dsmor_warp_active(out.ctypes.data if len(out) else None, len(out), w.ctypes.data)
    return out


# ---- output side of SurfelMap (SURVEY.md §8f row 4), restated in numpy.  cloud_points, mesh_vertices and
# ply_mesh_text are pinned byte for byte against the reference's own SurfelMap compiled in place (RefMap below,
# tests/test_refmap.py); pcd_text restates PCL's published PCD v0.7 ASCII layout (PCL is not vendored in the reference) ----
def cloud_points(local, min_update_times=5):
    """The local_surfels loop of publish_active_pointcloud / publish_all_pointcloud / save_cloud
    (surfel_map.cpp:1403-1412, :1429-1438, :1156-1166; `update_times < 5 -> continue`) and, with
    min_update_times=1, of publish_neighbor_pointcloud (:1291-1300): [n, 4] float32 x, y, z, intensity=color."""
    sel = local[local["update_times"] >= min_update_times]
    return np.stack([sel["px"], sel["py"], sel["pz"], sel["color"]], -1).astype(np.float32).reshape(-1, 4)


def mesh_vertices(surfels):
    """push_a_surfel (surfel_map.cpp:1175-1226) in float32, operation order as written: [n, 6, 6]."""
    f = np.float32
    n = len(surfels)
    col = surfels["color"].astype(np.int32).astype(f)                       # :1177
    p = np.stack([surfels["px"], surfels["py"], surfels["pz"]], -1).astype(f)
    nr = np.stack([surfels["nx"], surfels["ny"], surfels["nz"]], -1).astype(f)
    xd = np.stack([f(-1) * nr[:, 1], nr[:, 0], np.zeros(n, f)], -1)         # :1186-1188
    z = (xd[:, 0] * xd[:, 0] + xd[:, 1] * xd[:, 1]) + xd[:, 2] * xd[:, 2]   # normalize() :1189 (Eigen skips a zero vector)
    nz = z > 0
    with np.errstate(all="ignore"):
        xd[nz] = xd[nz] / np.sqrt(z[nz])[:, None]
    yd = np.stack([nr[:, 1] * xd[:, 2] - nr[:, 2] * xd[:, 1],               # cross :1191
                   nr[:, 2] * xd[:, 0] - nr[:, 0] * xd[:, 2],
                   nr[:, 0] * xd[:, 1] - nr[:, 1] * xd[:, 0]], -1)
    r = surfels["size"].astype(f)
    h_r = (r.astype(np.float64) * 0.5).astype(f)[:, None]                   # :1193
    t_r = (r.astype(np.float64) * 0.86603).astype(f)[:, None]               # :1194
    r = r[:, None]
    pts = [p - xd * h_r - yd * t_r, p + xd * h_r - yd * t_r, p - xd * r,    # :1196-1201
           p + xd * r, p - xd * h_r + yd * t_r, p + xd * h_r + yd * t_r]
    out = np.zeros((n, 6, 6), f)
    for k in range(6):
        out[:, k, :3] = pts[k]
        out[:, k, 3:] = col[:, None]
    return out


def _g(v, digits):
    return "%.*g" % (digits, float(v))


def ply_mesh_text(surfels):
    """SurfelMap::save_mesh (surfel_map.cpp:1229-1280): the exact bytes of the ASCII PLY (ostream default
    float format = %g with 6 digits; every vertex value is followed by a space)."""
    v = mesh_vertices(surfels).reshape(-1, 6)
    n = len(surfels)
    lines = ["ply", "format ascii 1.0", f"element vertex {n * 6}", "property float x", "property float y",
             "property float z", "property uchar red", "property uchar green", "property uchar blue",
             f"element face {n * 4}", "property list uchar int vertex_index", "end_header"]
    lines += ["".join(_g(x, 6) + " " for x in row) for row in v]
    for i in range(n):
        p1, p2, p3, p4, p5, p6 = (i * 6 + k for k in range(6))
        lines += [f"3 {p1} {p2} {p3}", f"3 {p2} {p4} {p3}", f"3 {p3} {p4} {p5}", f"3 {p5} {p4} {p6}"]
    return "\n".join(lines) + "\n"


def pcd_text(points):
    """pcl::io::savePCDFile(name, PointCloud<PointXYZI>) as called at surfel_map.cpp:1171 — PCL's ASCII writer
    (PCD v0.7 header, 8 significant digits, NaN spelled "nan"); PCL is not vendored in the reference tree."""
    pts = np.asarray(points, dtype=np.float32).reshape(-1, 4)
    n = len(pts)
    head = ["# .PCD v0.7 - Point Cloud Data file format", "VERSION 0.7", "FIELDS x y z intensity", "SIZE 4 4 4 4",
            "TYPE F F F F", "COUNT 1 1 1 1", f"WIDTH {n}", "HEIGHT 1", "VIEWPOINT 0 0 0 1 0 0 0", f"POINTS {n}", "DATA ascii"]
    body = [" ".join("nan" if np.isnan(x) else _g(x, 8) for x in row) for row in pts]
    return "\n".join(head + body) + "\n"


# ---- the reference's whole SurfelMap, compiled in place (oracle/ref_map_driver.cpp) ----
def have_refmap(b200=False):
    return have(RefMap.libname_b200 if b200 else RefMap.libname)


def pose_to_ros7(pose_colmajor16):
    """4x4 T_world<-cam (column-major, as the hot path takes it) -> the 7 numbers of a geometry_msgs::Pose
    (position xyz, orientation xyzw), i.e. what the pose feed publishes."""
    from scipy.spatial.transform import Rotation
    T = np.asarray(pose_colmajor16, np.float64).reshape(4, 4).T
    q = Rotation.from_matrix(T[:3, :3]).as_quat()  # x, y, z, w
    return np.array([T[0, 3], T[1, 3], T[2, 3], q[0], q[1], q[2], q[3]], np.float64)


class RefMap:
    """SurfelMap of the reference (surfel_fusion/src/surfel_map.cpp) behind oracle/ref_map_driver.cpp.
    b200=False: with the reference's own FusionFunctions (threads inlined: deterministic) -- the system-level oracle.
    b200=True : the same SurfelMap holding the product's dsm::FusionFunctions (INTEGRATION.md's patch); needs a GPU."""
    libname = "libdsm_refmap.so"
    libname_b200 = "libdsm_refmap_b200.so"

    def __init__(self, cam, drift_free_poses=10, b200=False):
        vp, ci, cf, cd = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_double
        self.lib = L = _lib(self.libname_b200 if b200 else self.libname)
        self.cam = cam
        L.dsmmap_create.restype = vp
        L.dsmmap_create.argtypes = [ci, ci, cf, cf, cf, cf, cf, cf, ci]
        L.dsmmap_destroy.argtypes = [vp]
        L.dsmmap_frame.argtypes = [vp, cd, vp, vp, vp, ci, ci, vp, ci, vp, ci]
        for name in ("dsmmap_num_local", "dsmmap_num_poses", "dsmmap_num_inactive_points"):
            getattr(L, name).argtypes = [vp]
        L.dsmmap_get_local.argtypes = [vp, vp]
        L.dsmmap_num_attached.argtypes = [vp, ci]
        L.dsmmap_get_attached.argtypes = [vp, ci, vp]
        L.dsmmap_get_inactive_points.argtypes = [vp, vp]
        L.dsmmap_published_points.argtypes = [ctypes.c_char_p, vp, ci]
        L.dsmmap_save_mesh.argtypes = [vp, ctypes.c_char_p]
        L.dsmmap_save_cloud.argtypes = [vp, ctypes.c_char_p]
        L.dsmmap_set_local.argtypes = [vp, vp, ci]
        L.dsmmap_warp_active.argtypes = [vp, vp]
        L.dsmmap_fuse_map.argtypes = [vp, vp, vp, vp, ci]
        L.dsmmap_move_add_surfels.argtypes = [vp, ci]
        L.dsmmap_publish_clouds.argtypes = [vp, ci]
        L.dsmmap_local_pose_indexs.argtypes = [vp, vp, ci]
        L.dsmmap_mesh_vertices.argtypes = [vp, vp, ci, vp]
        self.h = L.dsmmap_create(cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near, int(drift_free_poses))

    def close(self):
        if self.h:
            self.lib.dsmmap_destroy(self.h)
            self.h = None

    def frame(self, stamp, gray, depth, pose7, is_keyframe, reference_index, path7=(), loops=()):
        """One synchronised frame through the node's three callbacks (ros_node.cpp): pose feed, image, depth
        (gray=None: the pose feed callback only)."""
        gray = None if gray is None else np.ascontiguousarray(gray, np.uint8)
        depth = None if depth is None else np.ascontiguousarray(depth, np.float32)
        pose7 = np.ascontiguousarray(pose7, np.float64)
        path = np.ascontiguousarray(np.asarray(path7, np.float64).reshape(-1, 7))
        lp = np.ascontiguousarray(np.asarray(loops, np.int32).reshape(-1))
        self.lib.dsmmap_frame(self.h, float(stamp), None if gray is None else gray.ctypes.data,
                              None if depth is None else depth.ctypes.data, pose7.ctypes.data, int(is_keyframe),
                              int(reference_index), path.ctypes.data if len(path) else None, len(path),
                              lp.ctypes.data if len(lp) else None, len(lp) // 2)

    def local(self):
        out = np.zeros(self.lib.dsmmap_num_local(self.h), SURFEL_DTYPE)
        if len(out):
            self.lib.dsmmap_get_local(self.h, out.ctypes.data)
        return out

    def num_poses(self):
        return self.lib.dsmmap_num_poses(self.h)

    def attached(self, pose):
        out = np.zeros(self.lib.dsmmap_num_attached(self.h, pose), SURFEL_DTYPE)
        if len(out):
            self.lib.dsmmap_get_attached(self.h, pose, out.ctypes.data)
        return out

    def inactive_points(self):
        out = np.zeros((self.lib.dsmmap_num_inactive_points(self.h), 4), np.float32)
        if len(out):
            self.lib.dsmmap_get_inactive_points(self.h, out.ctypes.data)
        return out

    def published(self, topic, cap=4_000_000):
        """Last cloud on a topic ('active_pointcloud', 'inactive_pointcloud', 'pointcloud', 'neighbor_pointcloud',
        or 'file:<path>' for what save_cloud handed to the PCD writer) as [n, 4] float32, None if never published."""
        n = self.lib.dsmmap_published_points(topic.encode(), None, 0)
        if n < 0:
            return None
        out = np.zeros((max(n, 1), 4), np.float32)
        self.lib.dsmmap_published_points(topic.encode(), out.ctypes.data, n)
        return out[:n]

    def local_pose_indexs(self):
        out = np.zeros(4096, np.int32)
        n = self.lib.dsmmap_local_pose_indexs(self.h, out.ctypes.data, len(out))
        return out[:n].tolist()

    def save_mesh(self, path):
        self.lib.dsmmap_save_mesh(self.h, os.fsencode(path))

    def save_cloud(self, path):
        self.lib.dsmmap_save_cloud(self.h, os.fsencode(path))
        return self.published("file:" + str(path))

    # ---- the members one by one ----
    def set_local(self, surfels):
        s = np.ascontiguousarray(surfels, SURFEL_DTYPE)
        self.lib.dsmmap_set_local(self.h, s.ctypes.data if len(s) else None, len(s))

    def warp_active(self, W_colmajor):
        w = np.ascontiguousarray(W_colmajor, np.float32).reshape(16)
        self.lib.dsmmap_warp_active(self.h, w.ctypes.data)

    def fuse_map(self, gray, depth, pose_colmajor16, reference_index):
        gray = np.ascontiguousarray(gray, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        p = np.ascontiguousarray(pose_colmajor16, np.float32).reshape(16)
        self.lib.dsmmap_fuse_map(self.h, gray.ctypes.data, depth.ctypes.data, p.ctypes.data, int(reference_index))

    def move_add_surfels(self, reference_index):
        self.lib.dsmmap_move_add_surfels(self.h, int(reference_index))

    def publish_clouds(self, reference_index):
        self.lib.dsmmap_publish_clouds(self.h, int(reference_index))

    def mesh_vertices(self, surfels):
        s = np.ascontiguousarray(surfels, SURFEL_DTYPE)
        out = np.zeros((len(s), 6, 6), np.float32)
        if len(s):
            n = self.lib.dsmmap_mesh_vertices(self.h, s.ctypes.data, len(s), out.ctypes.data)
            assert n == 36 * len(s)
        return out


def have_reference():
    return have(RefSerial.libname)


# ---- comparison metrics (SURVEY.md §7 H5: norm-based, not per-component relative) ----
def surfel_errors(a, b):
    """Returns dict of max errors between two equally long SURFEL_DTYPE arrays."""
    assert len(a) == len(b)
    if len(a) == 0:
        return dict(pos=0.0, nrm=0.0, size=0.0, weight=0.0, color=0.0, int_mismatch=0)
    pa = np.stack([a["px"], a["py"], a["pz"]], -1).astype(np.float64)
    pb = np.stack([b["px"], b["py"], b["pz"]], -1).astype(np.float64)
    na = np.stack([a["nx"], a["ny"], a["nz"]], -1).astype(np.float64)
    nb = np.stack([b["nx"], b["ny"], b["nz"]], -1).astype(np.float64)
    pos = np.linalg.norm(pa - pb, axis=1) / np.maximum(np.linalg.norm(pb, axis=1), 1e-12)
    nrm = np.linalg.norm(na - nb, axis=1)
    size = np.abs(a["size"].astype(np.float64) - b["size"]) / np.maximum(np.abs(b["size"]), 1e-12)
    wgt = np.abs(a["weight"].astype(np.float64) - b["weight"]) / np.maximum(np.abs(b["weight"]), 1e-12)
    col = np.abs(a["color"].astype(np.float64) - b["color"])
    im = int(np.sum(a["update_times"] != b["update_times"]) + np.sum(a["last_update"] != b["last_update"]))
    return dict(pos=float(pos.max()), nrm=float(nrm.max()), size=float(size.max()),
                weight=float(wgt.max()), color=float(col.max()), int_mismatch=im)
