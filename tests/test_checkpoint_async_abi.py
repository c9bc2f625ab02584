"""CPU tests of the checkpoints that do not stop the stream (dsm_checkpoint_*, DESIGN.md §8.5): the calls are exported
and declared, and a null context, a null path or extra bytes without a buffer are refused without a device."""
import ctypes
import os

from densesurfelmapping_b200 import capi

CALLS = ["dsm_checkpoint_enable", "dsm_checkpoint_enqueue", "dsm_checkpoint_wait", "dsm_debug_checkpoint_drain_ctas"]


def test_calls_are_exported_and_declared():
    lib = capi.load_library()
    for name in CALLS:
        assert name in capi.EXPORTS and hasattr(lib, name), name


def test_null_arguments_are_invalid_without_a_device(tmp_path):
    L = capi.load_library()
    p = os.fsencode(tmp_path / "map.dsm")
    fin = ctypes.c_int(5)
    assert L.dsm_checkpoint_enable(None) == -1
    assert L.dsm_checkpoint_enqueue(None, p, None, 0) == -1
    assert L.dsm_checkpoint_enqueue(None, None, None, 0) == -1
    assert L.dsm_checkpoint_enqueue(None, p, None, 8) == -1          # extra bytes without a buffer
    assert L.dsm_checkpoint_wait(None, 1, ctypes.byref(fin)) == -1 and fin.value == 0
    assert L.dsm_checkpoint_wait(None, 0, None) == -1
    assert L.dsm_debug_checkpoint_drain_ctas(None, 16) == -1
    assert not os.path.exists(tmp_path / "map.dsm")
