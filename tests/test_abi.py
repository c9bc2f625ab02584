"""CPU tests: the C-ABI library loads and exports every symbol include/dsm.h declares, element
layouts match the reference PODs, and host-side error handling works without a GPU."""
import ctypes
import os
import re

import numpy as np

from densesurfelmapping_b200 import capi, elements, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "dsm.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dsm_[a-z_0-9]+)\s*\(", src)))


def test_header_and_binding_agree():
    decl = declared_functions()
    assert decl, "no functions parsed from include/dsm.h"
    assert sorted(capi.EXPORTS) == decl, (sorted(set(decl) - set(capi.EXPORTS)), sorted(set(capi.EXPORTS) - set(decl)))


def test_library_exports_every_declared_symbol():
    lib = capi.load_library()  # built by __graft_entry__.build(); raises if missing (no fallback)
    for name in declared_functions():
        assert hasattr(lib, name), f"libdsm_b200.so does not export {name}"
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dsm.h")).read()
    assert lib.dsm_version() == int(re.search(r"#define DSM_VERSION (\d+)", header).group(1))  # library built from this header
    assert lib.dsm_strerror(-2).decode().startswith("unsupported image shape")
    assert capi.kernel_names()[:3] == ["seed_init", "slic_assign_first", "slic_assign"]


def test_element_layouts_match_reference_pods():
    # elements.h:5-31 — 60-byte seed, 44-byte surfel
    assert elements.SEED_DTYPE.itemsize == 60 and elements.SURFEL_DTYPE.itemsize == 44
    assert elements.SEED_DTYPE.fields["fused"][1] == 48 and elements.SEED_DTYPE.fields["min_eigen_value"][1] == 52
    assert elements.SURFEL_DTYPE.fields["update_times"][1] == 36
    assert ctypes.sizeof(capi.DsmParams) == 40
    assert elements.num_seeds(1226, 370) == 7038 and elements.num_seeds(640, 480) == 4800


def test_create_fails_loudly_without_device_or_on_bad_shape():
    lib = capi.load_library()
    h = ctypes.c_void_p()
    bad = capi.DsmParams(645, 480, 1, 1, 1, 1, 30, 0.5, 1, 16)
    assert lib.dsm_create(ctypes.byref(bad), 0, None, ctypes.byref(h)) == -2  # DSM_E_SHAPE before touching CUDA
    assert lib.dsm_create(None, 0, None, ctypes.byref(h)) == -1
    import torch
    if not torch.cuda.is_available():
        ok = capi.DsmParams(640, 480, 525, 525, 319.5, 239.5, 30, 0.5, 1, 16)
        assert lib.dsm_create(ctypes.byref(ok), 0, None, ctypes.byref(h)) == -3  # DSM_E_NODEVICE: no CPU fallback
        assert not h.value


def test_synthetic_generator_is_deterministic():
    a = synth.make_frame(synth.VGA, 5, synth.pose_stream(5))
    b = synth.make_frame(synth.VGA, 5, synth.pose_stream(5))
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    assert a[0].dtype == np.uint8 and a[1].dtype == np.float32
    assert 0.005 < (a[1] == 0).mean() < 0.05  # ~1 % holes + the hole block
    p = synth.pose_stream(3).reshape(4, 4).T
    assert np.allclose(p[:3, :3] @ p[:3, :3].T, np.eye(3), atol=1e-6)


def test_float_bounds_for_double_literal_compares():
    """csrc/dsm_exact.cuh (used by every kernel file) replaces `(double)x < c` by `x < c_hi` (and `> c` by `> c_lo`) in hot loops;
    every F_<c>_HI / _LO constant must be the float neighbour of the double literal c, and the kernel files use exactly
    the constants the header defines."""
    csrc = os.path.join(ROOT, "densesurfelmapping_b200", "csrc")
    src = open(os.path.join(csrc, "dsm_exact.cuh")).read()
    found = re.findall(r"#define F_(\d+)p(\d+)_(HI|LO) __uint_as_float\(0x([0-9a-f]+)u\)", src)
    defined = {f"F_{ip}p{fp}_{kind}" for ip, fp, kind, _ in found}
    assert len(defined) == len(found) == len(re.findall(r"#define F_", src))  # every F_ macro parsed, none twice
    used = set()
    for name in os.listdir(csrc):
        if name.endswith(".cu"):
            used |= set(re.findall(r"\bF_\d+p\d+_(?:HI|LO)\b", open(os.path.join(csrc, name)).read()))
    assert used == defined, (sorted(used - defined), sorted(defined - used))
    for ip, fp, kind, hexv in found:
        c = float(f"{ip}.{fp}")
        f = np.array([int(hexv, 16)], dtype=np.uint32).view(np.float32)[0]
        if kind == "HI":  # smallest float >= c (c itself is not a float)
            assert float(f) > c and float(np.nextafter(f, np.float32(0))) < c, (c, kind, float(f))
        else:             # largest float <= c
            assert float(f) < c and float(np.nextafter(f, np.float32(10))) > c, (c, kind, float(f))
