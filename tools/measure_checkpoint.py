"""Time dsm_map_save and dsm_map_load (DESIGN.md §8.4) on one GPU at two map sizes.

  node      the size of tools/measure_node.py's end state: 81 Ki pool surfels, 47 Ki stored surfels in 80 segments
  large     1 Mi pool surfels, 4 Mi stored surfels in 1024 segments
The maps are built with dsm_pool_upload + dsm_inactive_load from seeded random surfels: the calls move plain records, so
their time depends on the sizes only.  The file goes to a temporary directory (--dir to choose its file system).
Reported per size, medians of --reps runs, with the card's name and power limit read in the same run:
  file_bytes, save_ms, load_ms, save_MBps, load_MBps (file bytes over wall time; both include the fsync / read of the file)
  readout_ms   the device part of a save: the synchronising reads of the pool, store and table (dsm_pool_download,
               dsm_inactive_download, dsm_inactive_segments) that a save makes before it writes.  The context's stream
               carries nothing else while they run; for the rest of the save the stream is idle, but the calling thread,
               which is the one that would enqueue the next frame, is still blocked, so save_ms is the stall a
               single-threaded node sees.
Usage: python tools/measure_checkpoint.py [--reps 5] [--dir DIR] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402

SIZES = {"node": (81 << 10, 47 << 10, 80), "large": (1 << 20, 4 << 20, 1024)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to measure on")
    name, power = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return name, power


def surfels(rng, n):
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
        s[f] = rng.standard_normal(n).astype(np.float32)
    s["update_times"] = rng.integers(1, 20, n)
    return s


def make_map(n_pool, n_store, n_seg, seed=7):
    rng = np.random.default_rng(seed)
    ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=n_pool)
    ctx.pool_upload(surfels(rng, n_pool))
    ctx.inactive_reserve(n_store)
    store = surfels(rng, n_store)
    cnt = np.full(n_seg, n_store // n_seg, np.int32)
    cnt[-1] += n_store - cnt.sum()
    ofs = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
    store["last_update"] = np.repeat(np.arange(n_seg, dtype=np.int32), cnt)
    ctx.inactive_load(store, np.stack([np.arange(n_seg, dtype=np.int32), ofs, cnt], 1))
    return ctx


def measure(name, reps, d):
    n_pool, n_store, n_seg = SIZES[name]
    ctx = make_map(n_pool, n_store, n_seg)
    path = os.path.join(d, f"{name}.dsm")
    save, load, readout = [], [], []
    want = (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes())
    for _ in range(reps + 1):            # the first round warms the allocator and the page cache
        a = time.perf_counter()
        ctx.pool_download(), ctx.inactive_download(-1), ctx.inactive_segments()
        b = time.perf_counter()
        ctx.map_save(path)
        c = time.perf_counter()
        ctx.map_load(path)
        e = time.perf_counter()
        readout.append((b - a) * 1e3)
        save.append((c - b) * 1e3)
        load.append((e - c) * 1e3)
    assert (ctx.pool_download().tobytes(), ctx.inactive_download(-1).tobytes()) == want
    size = os.path.getsize(path)
    os.remove(path)
    ctx.close()
    med = lambda x: float(np.median(x[1:]))  # noqa: E731
    return {"pool_surfels": n_pool, "store_surfels": n_store, "segments": n_seg, "file_bytes": size,
            "save_ms": med(save), "load_ms": med(load), "readout_ms": med(readout),
            "save_MBps": size / med(save) / 1e3, "load_MBps": size / med(load) / 1e3,
            "save_ms_all": save[1:], "load_ms_all": load[1:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power}
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        for size in SIZES:
            res[size] = measure(size, a.reps, d)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_checkpoint.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
