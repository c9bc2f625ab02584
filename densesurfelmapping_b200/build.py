"""Builds the product library ``densesurfelmapping_b200/libdsm_b200.so`` in-tree with nvcc for
sm_90a.  -fmad=false is part of the exactness contract (see csrc/dsm_kernels.cu header)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdsm_b200.so")
SOURCES = ["dsm_kernels.cu", "dsm_tile.cu", "dsm_capi.cu", "dsm_comm.cu", "dsm_io.cpp", "dsm_field.cu", "dsm_frontier.cu", "dsm_reach.cu", "dsm_gain.cu", "dsm_tour.cu", "dsm_viewpoint.cu", "dsm_trajectory.cu", "dsm_heading.cu", "dsm_terrain.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off", "-shared", "-cudart", "shared", "-ldl",
]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "dsm.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return LIB
    tmp = LIB + ".tmp"  # linked next to the target and renamed: a concurrent reader (gpurun snapshot) never sees a half-written library
    cmd = [_nvcc()] + NVCC_FLAGS + list(extra) + ["-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(" ".join(cmd))
        print(r.stdout)
        print(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed")
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    import sys
    build(force=True, verbose=True, extra=["-Xptxas", "-v"] if "-v" in sys.argv else [])
