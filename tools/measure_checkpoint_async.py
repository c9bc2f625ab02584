"""Measure the checkpoints that do not stop the stream (dsm_checkpoint_*, DESIGN.md §8.5) on one GPU.

  kernels   k_map_snapshot and k_map_drain device times (torch.profiler, CUDA activities), medians of --reps checkpoints,
            at the two sizes of tools/measure_checkpoint.py (node: 81 Ki pool + 47 Ki stored surfels; large: 1 Mi + 4 Mi),
            with the snapshot's model rate (2 x 44 B per surfel + 28 B per segment over its time, against 3.35 TB/s)
            and the drain's rate over PCIe (the live bytes it moves over its time)
  drain     k_map_drain at the large size for several CTA counts (dsm_debug_checkpoint_drain_ctas)
  durable   wall time from dsm_checkpoint_enqueue to the dsm_checkpoint_wait that reports the file on the disk, beside
            dsm_map_save of the same map, and the enqueue call alone
  node      tools/measure_node.py's drive (320 frames) through tools/measure_checkpoint_async.cpp, no synchronisation per
            frame, ms per frame in four modes alternating for --rounds rounds: no checkpoint; save_state_async once 20
            frames have passed, skipped while the previous one is written (INTEGRATION.md section 4); the blocking
            save_state every 20 frames; save_state_async every 20 frames, waiting for a previous one still in flight
            (with the host time spent in those waits); and the host time inside the save calls
The card's name and power limit are read in the same run.  Files go to a temporary directory.
Usage: python tools/measure_checkpoint_async.py [--reps 5] [--rounds 3] [--out DIR]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from measure_drive import SIZES, build_harness, card, images, kernel_us, make_map, messages, run_harness, write_drive  # noqa: E402

HBM_TBPS = 3.35
DRAIN_CTAS = (4, 8, 16, 32, 66, 132)


def live_bytes(n_pool, n_store, n_seg):
    line = lambda b: (b + 127) // 128 * 128  # noqa: E731
    return 128 + line(44 * n_pool) + line(44 * n_store) + line(12 * n_seg)


def measure_size(name, reps, d):
    n_pool, n_store, n_seg = SIZES[name]
    ctx = make_map(n_pool, n_store, n_seg)
    ctx.checkpoint_enable()
    path = os.path.join(d, f"{name}.dsm")
    ctx.checkpoint_enqueue(path)
    ctx.checkpoint_wait()

    def ckpts():
        for _ in range(reps):
            ctx.checkpoint_enqueue(path)
            ctx.checkpoint_wait()
    t = kernel_us(ckpts, ("k_map_snapshot", "k_map_drain"))
    snap, drain = float(np.median(t["k_map_snapshot"])), float(np.median(t["k_map_drain"]))
    moved = 2 * 44 * (n_pool + n_store) + 28 * n_seg
    res = {"pool_surfels": n_pool, "store_surfels": n_store, "segments": n_seg, "snapshot_us": snap,
           "snapshot_model_bytes": moved, "snapshot_TBps": moved / snap / 1e6, "snapshot_of_peak": moved / snap / 1e6 / HBM_TBPS,
           "drain_us": drain, "drain_bytes": live_bytes(n_pool, n_store, n_seg),
           "drain_GBps": live_bytes(n_pool, n_store, n_seg) / drain / 1e3}
    enq, dur, sync = [], [], []
    for _ in range(reps):
        a = time.perf_counter()
        ctx.checkpoint_enqueue(path)
        b = time.perf_counter()
        ctx.checkpoint_wait()
        c = time.perf_counter()
        ctx.map_save(path)
        e = time.perf_counter()
        enq.append((b - a) * 1e3)
        dur.append((c - a) * 1e3)
        sync.append((e - c) * 1e3)
    res.update({"file_bytes": os.path.getsize(path), "enqueue_ms": float(np.median(enq)), "enqueue_to_durable_ms": float(np.median(dur)),
                "map_save_ms": float(np.median(sync)), "enqueue_to_durable_ms_all": dur, "map_save_ms_all": sync})
    if name == "large":
        sweep = {}
        for n in DRAIN_CTAS:
            assert ctx.lib.dsm_debug_checkpoint_drain_ctas(ctx.h, n) == 0
            t = kernel_us(ckpts, ("k_map_drain",))
            us = float(np.median(t["k_map_drain"]))
            sweep[str(n)] = {"drain_us": us, "drain_GBps": res["drain_bytes"] / us / 1e3}
        res["drain_ctas"] = sweep
    os.remove(path)
    ctx.close()
    return res


def node_drive(tmp, rounds, frames, every=20):
    exe = build_harness(tmp, "measure_checkpoint_async")
    ff, fs = write_drive(tmp, images(), messages(frames))
    out = {"none": [], "save_state_async": [], "save_state": [], "save_state_async_waiting": []}
    last, skipped, wait_ms, call_ms = {}, {k: [] for k in out}, {k: [] for k in out}, {k: [] for k in out}
    for _ in range(rounds):
        for mode, key in enumerate(out):
            last[key] = run_harness(exe, ff, fs, [mode, every, tmp])
            out[key].append(last[key]["ms_per_frame"])
            skipped[key].append(last[key]["skipped"])
            wait_ms[key].append(last[key]["wait_ms"])
            call_ms[key].append(last[key]["save_call_ms"])
    return {"frames": frames, "every": every, "ms_per_frame": out, "saves": {k: v["saves"] for k, v in last.items()},
            "skipped": skipped, "wait_ms": wait_ms, "save_call_ms": call_ms,
            "store_surfels": last["none"]["store_surfels"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power}
    with tempfile.TemporaryDirectory() as d:
        for size in SIZES:
            res[size] = measure_size(size, a.reps, d)
        res["node_drive"] = node_drive(d, a.rounds, a.frames)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_checkpoint_async.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
