"""Measure incremental checkpoints (dsm_checkpoint_enqueue_incremental, DESIGN.md §8.6) on one GPU.

  large     1 Mi pool + 4 Mi stored surfels in 1024 segments (tools/measure_checkpoint.py's large map; the pool's surfels
            spread over 64 keyframes), --reps checkpoints for each change pattern between two checkpoints:
              none      nothing changes: a record holds the table, the header and no chunk
              retire    dsm_inactive_retire of one pool keyframe (~16 Ki surfels): the store grows at its tail, and the
                        pool loses that keyframe's surfels
              warp_all  dsm_pool_transform plus dsm_inactive_transform of every stored keyframe: every chunk changes (the
                        worst case; the journal outgrows its base every second record, so bases and records alternate)
            per pattern: k_map_delta and k_map_drain_delta device times (torch.profiler, medians), the record's bytes and
            changed chunks, and the wall time from the enqueue to the dsm_checkpoint_wait that reports the record on the
            disk; then, in the same job, the same pattern with the full dsm_checkpoint_enqueue (k_map_snapshot,
            k_map_drain, enqueue to durable file) for comparison
  node      tools/measure_node.py's drive (320 frames) through tools/measure_checkpoint_journal.cpp, a checkpoint once 20
            frames have passed (skipped while the previous one is written), ms per frame in three modes alternating for
            --rounds rounds: no checkpoint, save_state_async, save_state_incremental; and the bytes each save wrote
The card's name and power limit are read in the same run.  Files go to a temporary directory.
Usage: python tools/measure_checkpoint_journal.py [--reps 5] [--rounds 3] [--out DIR]"""
import argparse
import json
import os
import struct
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from densesurfelmapping_b200 import capi, synth  # noqa: E402
from measure_drive import build_harness, card, images, kernel_us, messages, run_harness, surfels, write_drive  # noqa: E402

N_POOL, N_STORE, N_SEG, POOL_KEYS = 1 << 20, 4 << 20, 1024, 64


def large_map():
    rng = np.random.default_rng(7)
    ctx = capi.Context(synth.KITTI, max_batch=2, max_local_surfels=N_POOL)
    pool = surfels(rng, N_POOL)
    pool["last_update"] = N_SEG + rng.integers(0, POOL_KEYS, N_POOL)
    ctx.pool_upload(pool)
    ctx.inactive_reserve(N_STORE + 2 * N_POOL)         # a retirement needs room for the whole pool
    store = surfels(rng, N_STORE)
    cnt = np.full(N_SEG, N_STORE // N_SEG, np.int32)
    ofs = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
    store["last_update"] = np.repeat(np.arange(N_SEG, dtype=np.int32), cnt)
    ctx.inactive_load(store, np.stack([np.arange(N_SEG, dtype=np.int32), ofs, cnt], 1))
    ctx.checkpoint_enable()
    return ctx


def change(ctx, pattern, i):
    if pattern == "retire":
        ctx.inactive_retire(N_SEG + i % POOL_KEYS)
    elif pattern == "warp_all":
        w = np.eye(4, dtype=np.float32)
        w[0, 3] = 1e-3 * (i + 1)
        ctx.pool_transform(w)
        for kf in sorted(set(ctx.inactive_segments()[:, 0].tolist())):
            ctx.inactive_transform(kf, w)


def measure_pattern(pattern, reps, d):
    ctx = large_map()
    path = os.path.join(d, "large.dsm")
    jp = path + ".journal"
    ctx.checkpoint_enqueue_incremental(path)            # the base
    ctx.checkpoint_wait()
    res = {"records": [], "bases": 0}
    for i in range(reps):
        change(ctx, pattern, i)
        before = os.path.getsize(jp)
        t = {}

        def one():
            a = time.perf_counter()
            ctx.checkpoint_enqueue_incremental(path)
            ctx.checkpoint_wait()
            t["ms"] = (time.perf_counter() - a) * 1e3
        k = kernel_us(one, ("k_map_delta", "k_map_drain_delta", "k_map_snapshot", "k_map_drain"))
        after = os.path.getsize(jp)
        if k["k_map_delta"]:
            j = open(jp, "rb").read()[before:]
            kp, ks = struct.unpack_from("<ii", j, 20)
            res["records"].append({"bytes": after - before, "pool_chunks": kp, "store_chunks": ks, "enqueue_to_durable_ms": t["ms"],
                                   "k_map_delta_us": k["k_map_delta"][0], "k_map_drain_delta_us": k["k_map_drain_delta"][0]})
        else:
            res["bases"] += 1
    res["base_bytes"] = os.path.getsize(path)
    # the same pattern with whole files
    full = []
    for i in range(reps):
        change(ctx, pattern, reps + i)
        t = {}

        def one():
            a = time.perf_counter()
            ctx.checkpoint_enqueue(os.path.join(d, "full.dsm"))
            ctx.checkpoint_wait()
            t["ms"] = (time.perf_counter() - a) * 1e3
        k = kernel_us(one, ("k_map_snapshot", "k_map_drain"))
        full.append({"bytes": os.path.getsize(os.path.join(d, "full.dsm")), "enqueue_to_durable_ms": t["ms"],
                     "k_map_snapshot_us": k["k_map_snapshot"][0], "k_map_drain_us": k["k_map_drain"][0]})
    res["full"] = full
    med = lambda xs: float(np.median(xs)) if xs else None  # noqa: E731
    r = res["records"]
    res["median"] = {"record_bytes": med([x["bytes"] for x in r]), "record_enqueue_to_durable_ms": med([x["enqueue_to_durable_ms"] for x in r]),
                     "k_map_delta_us": med([x["k_map_delta_us"] for x in r]), "k_map_drain_delta_us": med([x["k_map_drain_delta_us"] for x in r]),
                     "full_bytes": med([x["bytes"] for x in full]), "full_enqueue_to_durable_ms": med([x["enqueue_to_durable_ms"] for x in full]),
                     "k_map_snapshot_us": med([x["k_map_snapshot_us"] for x in full]), "k_map_drain_us": med([x["k_map_drain_us"] for x in full])}
    ctx.close()
    for f in os.listdir(d):
        os.remove(os.path.join(d, f))
    return res


def node_drive(tmp, rounds, frames, every=20):
    exe = build_harness(tmp, "measure_checkpoint_journal")
    ff, fs = write_drive(tmp, images(), messages(frames))
    out = {"none": [], "save_state_async": [], "save_state_incremental": []}
    last = {}
    for _ in range(rounds):
        for mode, key in enumerate(out):
            last[key] = run_harness(exe, ff, fs, [mode, every, tmp])
            out[key].append(last[key]["ms_per_frame"])
    return {"frames": frames, "every": every, "ms_per_frame": out,
            "saves": {k: {"bytes": v["bytes"], "base": v["base"], "skipped": v["skipped"]} for k, v in last.items()}}


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
        for pattern in ("none", "retire", "warp_all"):
            res[pattern] = measure_pattern(pattern, a.reps, d)
        res["node_drive"] = node_drive(d, a.rounds, a.frames)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_checkpoint_journal.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
