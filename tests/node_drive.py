"""Driving the node drivers of tests/cpp: the drive of ORB messages, the message script the drivers read, the reader of
their out.bin, and building and running a driver."""
import atexit
import functools
import os
import shutil
import struct
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "densesurfelmapping_b200")


@functools.lru_cache(maxsize=None)
def _bin_dir():
    d = tempfile.mkdtemp(prefix="dsm_cpp_adapter_")
    atexit.register(shutil.rmtree, d, True)
    return d


@functools.lru_cache(maxsize=None)
def build_adapter(name="adapter_main"):
    """tests/cpp/<name>.cpp compiled once per session, outside the tree (the checkout may be read-only)."""
    src = os.path.join(ROOT, "tests", "cpp", name + ".cpp")
    out = os.path.join(_bin_dir(), name)
    cmd = ["g++", "-std=c++11", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle", "shim"), src,
           "-o", out, "-L", PKG, "-ldsm_b200", f"-Wl,-rpath,{PKG}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def cam_args(cam):
    """The camera arguments every driver starts with: W H fx fy cx cy far near."""
    return [str(cam.width), str(cam.height)] + [repr(float(v)) for v in (cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near)]


def correction(k):
    """The k-th loop correction the ORB side applies to its whole path: a small yaw and shift, none for k = 0."""
    M = np.eye(4)
    if k:
        M[:3, :3] = Rotation.from_euler("y", 0.7 * k, degrees=True).as_matrix()
        M[:3, 3] = [0.05 * k, -0.02 * k, 0.03 * k]
    return M


def ros7(M):
    q = Rotation.from_matrix(M[:3, :3]).as_quat()
    return np.array([M[0, 3], M[1, 3], M[2, 3], q[0], q[1], q[2], q[3]], np.float64)


def drive(n_frames=30):
    """The message sequence of a drive, one ORB message per frame: [(stamp, is_kf, reference, pose7, path7, loops)].
    A keyframe every other frame, referenced to the newest keyframe; frame 9 closes a loop to keyframe 0 (it re-enters
    the window); frames 12-13 refer back to keyframe 1 (keyframes leave, old ones return, then leave again); from frame
    16 the ORB side corrects every pose (the loop path moves every pose); at frames 21-22 the path leaves out the two
    newest keyframes and at 22 a new correction comes in (the last correction is carried to the uncovered poses)."""
    out, kf_frames, last_kf = [], [], 0
    for t in range(n_frames):
        P = np.asarray(synth.pose_stream(t), np.float64).reshape(4, 4).T
        k = 0 if t < 16 else (1 if t < 22 else 2)
        C = correction(k)
        is_kf = t % 2 == 0
        ref = 1 if t in (12, 13) else (last_kf if t else 0)
        covered = kf_frames[:-2] if t in (21, 22) else kf_frames
        path = [ros7(C @ np.asarray(synth.pose_stream(f), np.float64).reshape(4, 4).T) for f in covered]
        out.append((100.0 + 0.1 * t, is_kf, ref, ros7(C @ P), path, [4, 0] if t == 9 else []))
        if is_kf:
            kf_frames.append(t)
            last_kf = len(kf_frames) - 1
    return out


# ---- the message script of tests/cpp/node_main.cpp and its dumps ----
class Script:
    def __init__(self):
        self.b = bytearray()

    def orb(self, stamp, is_kf, ref, pose7, path7, loops):
        path = np.asarray(path7, np.float64).reshape(-1, 7)
        self.b += struct.pack("<idii", 0, stamp, int(is_kf), int(ref)) + np.asarray(pose7, np.float64).tobytes()
        self.b += struct.pack("<i", len(path)) + path.tobytes()
        self.b += struct.pack("<i", len(loops) // 2) + np.asarray(loops, np.int32).tobytes()

    def images(self, stamp, gray, depth):
        self.b += struct.pack("<id", 1, stamp) + np.ascontiguousarray(gray, np.uint8).tobytes()
        self.b += struct.pack("<id", 2, stamp) + np.ascontiguousarray(depth, np.float32).tobytes()

    def image(self, stamp, gray):
        self.b += struct.pack("<id", 1, stamp) + np.ascontiguousarray(gray, np.uint8).tobytes()

    def depth(self, stamp, depth):
        self.b += struct.pack("<id", 2, stamp) + np.ascontiguousarray(depth, np.float32).tobytes()

    def dump(self, poses=True, map_state=False, neighbor_ref=0):
        self.b += struct.pack("<iii", 3, int(poses) | (2 * int(map_state)), int(neighbor_ref))

    def save(self, mesh, cloud):
        a, c = os.fsencode(mesh), os.fsencode(cloud)
        self.b += struct.pack("<ii", 4, len(a)) + a + struct.pack("<i", len(c)) + c


def node_script(cam, n):
    """The script of drive(n): per frame its orb message, then the image and depth of a seeded frame at its pose."""
    sc = Script()
    for t, (stamp, is_kf, ref, p7, path, loops) in enumerate(drive(n)):
        sc.orb(stamp, is_kf, ref, p7, path, loops)
        sc.images(stamp, *synth.make_frame(cam, 3000 + t, synth.pose_stream(t)))
    return sc


class Reader:
    def __init__(self, raw):
        self.raw, self.o = raw, 0

    def take(self, dtype, n):
        a = np.frombuffer(self.raw, dtype, n, self.o)
        self.o += a.nbytes
        return a

    def i(self):
        return int(self.take(np.int32, 1)[0])

    def lst(self, dtype=np.int32):
        return self.take(dtype, self.i())


def read_dumps(raw, kinds):
    """kinds: the (poses, map_state) flags of each dump, in order."""
    r, out = Reader(raw), []
    for poses, map_state in kinds:
        d = {"rc": r.i()}
        if poses:
            n = r.i()
            d["cam"], d["loop"], d["links"] = [], [], []
            for _ in range(n):
                d["cam"].append(r.take(np.float64, 7))
                d["loop"].append(r.take(np.float64, 7))
                d["links"].append(r.lst().tolist())
            d["local"] = r.lst().tolist()
            ref = r.i()
            pose = r.take(np.float32, 16)
            rem, add = r.lst().tolist(), r.lst().tolist()
            d["pending"] = None if ref < 0 else (ref, pose, rem, add)
            d["driftfree"], d["lists"] = [], []
            for _ in range(n):
                d["driftfree"].append(r.lst().tolist())
                d["lists"].append((r.lst().tolist(), r.lst().tolist()))
            d["warp"] = [(r.i(), r.take(np.float32, 16)) for _ in range(r.i())]
            d["fuse_pose"] = r.take(np.float64, 7)
        if map_state:
            d["map_rc"] = r.i()
            d["local_surfels"] = r.lst(SURFEL_DTYPE)
            d["attached"] = [r.lst(SURFEL_DTYPE) for _ in range(len(d["cam"]))]   # map dumps come with the poses
            d["active"], d["inactive"], d["all"], d["neighbor"] = (r.lst(POINT_DTYPE) for _ in range(4))
        out.append(d)
    assert r.o == len(raw)
    return out


def _run(name, tmp, cam, script, args, tag, after):
    fin, fout = os.path.join(tmp, f"script{tag}.bin"), os.path.join(tmp, f"out{tag}.bin")
    with open(fin, "wb") as f:
        f.write(bytes(script.b))
    argv = [build_adapter(name)] + cam_args(cam) + [str(a) for a in args] + [fin, fout] + [str(a) for a in after]
    r = subprocess.run(argv, capture_output=True, text=True)
    return r, fout


def run_driver(name, tmp, cam, script, args, tag="", after=()):
    """Runs tests/cpp/<name>.cpp as `name W H fx fy cx cy far near *args in.bin out.bin *after` on the script, written to
    <tmp>/script<tag>.bin, asserts that it exits with 0 and returns a Reader over <tmp>/out<tag>.bin."""
    r, fout = _run(name, tmp, cam, script, args, tag, after)
    assert r.returncode == 0, r.stderr
    return Reader(open(fout, "rb").read())


def run_node(tmp, cam, script, drift_free_poses, device=-1, max_local=1 << 20, max_inactive=1 << 21, rgbd=False, check=True):
    r, fout = _run("node_main", tmp, cam, script, [drift_free_poses, device, max_local, max_inactive, int(rgbd)], "", ())
    if check:
        assert r.returncode == 0, r.stderr
    return r, open(fout, "rb").read() if os.path.exists(fout) else b""
