"""The checkpoint files as the GPU-resident map writes them (DESIGN.md §8.4, §8.6), read and written with numpy: the
version-1 file of dsm_map_save and the record headers of its journal."""
import numpy as np

from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE

HEADER = np.dtype([("magic", "S8"), ("format", "<u4"), ("version", "<i4"), ("width", "<i4"), ("height", "<i4"),
                   ("geometry", "<f4", 6), ("constants", "<f8", 4), ("n_pool", "<i4"), ("n_store", "<i4"),
                   ("n_segments", "<i4"), ("zero", "<i4"), ("extra_bytes", "<u8")])
MAGIC, FORMAT = b"DSMMAP", 1
JHEADER = np.dtype([("magic", "S8"), ("format", "<u4"), ("zero", "<u4"), ("base", "<u8")])
RHEADER = np.dtype([("sequence", "<u8"), ("n_pool", "<i4"), ("n_store", "<i4"), ("n_segments", "<i4"), ("k_pool", "<i4"),
                    ("k_store", "<i4"), ("zero", "<u4"), ("extra_bytes", "<u8")])
CHUNK = 256   # surfels per journal chunk


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


def changed(old, new):
    """Indices of the 256-surfel chunks of `new` that differ from `old` or reach beyond its size (what k_map_delta flags)."""
    out = []
    for c in range((len(new) + CHUNK - 1) // CHUNK):
        a, b = c * CHUNK, min(len(new), c * CHUNK + CHUNK)
        if b > len(old) or old[a:b].tobytes() != new[a:b].tobytes():
            out.append(c)
    return out
