"""CPU tests of the map checkpoint (dsm_map_save / dsm_map_load / dsm_map_peek, DESIGN.md §8.4): the calls are exported,
reject a null context or path without a device, and the library reads a file this module writes with numpy from the
documented layout -- extra bytes, segment table and checksum -- and refuses a truncated, corrupted or foreign one."""
import ctypes
import os

import numpy as np

from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE

HEADER = np.dtype([("magic", "S8"), ("format", "<u4"), ("version", "<i4"), ("width", "<i4"), ("height", "<i4"),
                   ("geometry", "<f4", 6), ("constants", "<f8", 4), ("n_pool", "<i4"), ("n_store", "<i4"),
                   ("n_segments", "<i4"), ("zero", "<i4"), ("extra_bytes", "<u8")])
MAGIC, FORMAT = b"DSMMAP", 1
CALLS = ["dsm_inactive_segments", "dsm_inactive_load", "dsm_map_save", "dsm_map_load", "dsm_map_peek"]


def fnv1a64(data):
    h = 0xcbf29ce484222325
    for b in bytes(data):
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def parse(raw):
    """(header, pool, store, table [n, 3], extra, checksum ok) of a checkpoint file's bytes."""
    h = np.frombuffer(raw, HEADER, 1)[0]
    o = HEADER.itemsize
    pool = np.frombuffer(raw, SURFEL_DTYPE, int(h["n_pool"]), o)
    o += pool.nbytes
    store = np.frombuffer(raw, SURFEL_DTYPE, int(h["n_store"]), o)
    o += store.nbytes
    table = np.frombuffer(raw, np.int32, 3 * int(h["n_segments"]), o).reshape(-1, 3)
    o += table.nbytes
    extra = raw[o:o + int(h["extra_bytes"])]
    o += len(extra)
    assert o + 8 == len(raw)
    ok = np.frombuffer(raw, "<u8", 1, o)[0] == fnv1a64(raw[:o])
    return h, pool, store, table, extra, bool(ok)


def build(pool, store, table, extra, width=320, height=240, geometry=(262.5, 262.5, 159.5, 119.5, 30.0, 0.5),
          constants=capi.CONSTANTS_DRIVE):
    h = np.zeros(1, HEADER)
    h["magic"], h["format"], h["version"] = MAGIC, FORMAT, capi.load_library().dsm_version()
    h["width"], h["height"], h["geometry"], h["constants"] = width, height, geometry, constants
    h["n_pool"], h["n_store"], h["n_segments"], h["extra_bytes"] = len(pool), len(store), len(table), len(extra)
    body = h.tobytes() + pool.tobytes() + store.tobytes() + np.asarray(table, np.int32).tobytes() + bytes(extra)
    return body + np.array([fnv1a64(body)], "<u8").tobytes()


def sample():
    pool = np.zeros(5, SURFEL_DTYPE)
    pool["px"] = np.arange(5)
    pool["update_times"] = [1, 0, 3, 7, 2]
    store = np.zeros(4, SURFEL_DTYPE)
    store["update_times"], store["last_update"] = 1, [3, 3, 1, 3]
    return pool, store, np.array([[3, 0, 2], [1, 2, 1], [3, 3, 1]], np.int32), b"node section \x00\x01"


def test_calls_are_exported_and_declared():
    lib = capi.load_library()
    for name in CALLS:
        assert name in capi.EXPORTS and hasattr(lib, name), name


def test_null_context_or_path_is_invalid_without_a_device(tmp_path):
    L = capi.load_library()
    n, sz = ctypes.c_int(0), ctypes.c_size_t(0)
    p = os.fsencode(tmp_path / "map.dsm")
    assert L.dsm_inactive_segments(None, None, 0, ctypes.byref(n)) == -1
    assert L.dsm_inactive_load(None, None, 0, None, 0) == -1
    assert L.dsm_map_save(None, p, None, 0) == -1
    assert L.dsm_map_load(None, p, None, 0, ctypes.byref(sz)) == -1
    assert L.dsm_map_peek(None, None, 0, None, None, 0, None) == -1
    assert not os.path.exists(tmp_path / "map.dsm")


def test_peek_reads_the_documented_layout(tmp_path):
    pool, store, table, extra = sample()
    path = tmp_path / "map.dsm"
    path.write_bytes(build(pool, store, table, extra))
    got_extra, got_table = capi.map_peek(path)
    assert got_extra == extra and got_table.tolist() == table.tolist()
    h, p2, s2, t2, e2, ok = parse(path.read_bytes())
    assert ok and p2.tobytes() == pool.tobytes() and s2.tobytes() == store.tobytes() and e2 == extra
    # empty sections
    path.write_bytes(build(pool[:0], store[:0], table[:0], b""))
    assert capi.map_peek(path)[0] == b"" and len(capi.map_peek(path)[1]) == 0


def test_peek_refuses_damaged_and_foreign_files(tmp_path):
    pool, store, table, extra = sample()
    raw = build(pool, store, table, extra)
    L = capi.load_library()

    def peek(data):
        path = tmp_path / "x.dsm"
        path.write_bytes(data)
        return L.dsm_map_peek(os.fsencode(path), None, 0, None, None, 0, None)

    assert peek(raw) == 0
    assert peek(raw[:-1]) == -9                            # truncated
    assert peek(raw[:HEADER.itemsize + 50]) == -9
    assert peek(raw[:10]) == -9
    flipped = bytearray(raw)
    flipped[HEADER.itemsize + 7] ^= 0x10                   # one payload byte
    assert peek(bytes(flipped)) == -9
    wrong = bytearray(raw)
    wrong[0:1] = b"X"                                      # magic
    assert peek(bytes(wrong)) == -1
    newer = bytearray(raw)
    newer[8] = FORMAT + 1                                  # format version
    assert peek(bytes(newer)) == -1
    assert L.dsm_map_peek(os.fsencode(tmp_path / "missing.dsm"), None, 0, None, None, 0, None) == -9


def test_peek_copies_at_most_cap(tmp_path):
    pool, store, table, extra = sample()
    path = tmp_path / "map.dsm"
    path.write_bytes(build(pool, store, table, extra))
    L = capi.load_library()
    buf, seg = ctypes.create_string_buffer(4), np.zeros((1, 3), np.int32)
    ne, ns = ctypes.c_size_t(0), ctypes.c_int(0)
    assert L.dsm_map_peek(os.fsencode(path), buf, 4, ctypes.byref(ne), seg.ctypes.data, 1, ctypes.byref(ns)) == 0
    assert ne.value == len(extra) and ns.value == 3 and buf.raw == extra[:4] and seg[0].tolist() == table[0].tolist()
