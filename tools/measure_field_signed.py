"""Measure the signed distance field (dsm_field_signed_enable, DESIGN.md §8.16).

1. Latency: host clock from dsm_field_enqueue (host copy) or dsm_field_enqueue_resident to the end of dsm_field_wait,
   on an idle stream, for two contexts over the same map, one without and one with the signed grid, alternating
   --rounds times (--reps requests each).  The map is tools/measure_field.py's: a store of --store surfels spread over
   the box, voxel 0.1 m.
2. Kernels (torch.profiler, CUDA activities, --launches resident requests with the signed grid): the three new passes,
   k_field_rows<false, true>, the second k_field_lines<false> and k_field_lines_signed, against the first three.
The card's name and power limit are read in the same run.  Fails without a GPU.
Usage: python tools/measure_field_signed.py [--grids 200x200x60 320x320x40 512x512x64] [--out DIR]"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from measure_drive import card, spread  # noqa: E402
from measure_field import stored_context  # noqa: E402


def latency(ctx, host_copy, reps):
    lib, h = ctx.lib, ctx.h
    c = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    fn = lib.dsm_field_enqueue if host_copy else lib.dsm_field_enqueue_resident
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        assert fn(h, c, 5) == 0
        assert lib.dsm_field_wait(h, None, None, None) == 0
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def kernels(ctx, launches):
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib, h = ctx.lib, ctx.h
    c = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for _ in range(5):
        assert lib.dsm_field_enqueue_resident(h, c, 5) == 0 and lib.dsm_field_wait(h, None, None, None) == 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            assert lib.dsm_field_enqueue_resident(h, c, 5) == 0
            assert lib.dsm_field_wait(h, None, None, None) == 0
        torch.cuda.synchronize()
    out = {}
    for name, key, per in (("rows", "k_field_rows<false, false>", 1), ("rows_complement", "k_field_rows<false, true>", 1),
                           ("y_passes", "k_field_lines<false>", 2), ("z_pass", "k_field_lines<true>", 1),
                           ("z_pass_signed", "k_field_lines_signed", 1)):
        rows = [k for k in prof.key_averages() if key in k.key]
        count = sum(k.count for k in rows)
        if count != per * launches:
            raise RuntimeError(f"profiler saw {count} launches of {key}, expected {per * launches}")
        out[name] = {"us_per_request": sum(k.device_time_total for k in rows) / launches, "launches_per_request": per}
    y = out["y_passes"]["us_per_request"] / 2
    out["unsigned_passes_us"] = out["rows"]["us_per_request"] + y + out["z_pass"]["us_per_request"]
    out["signed_passes_us"] = out["rows_complement"]["us_per_request"] + y + out["z_pass_signed"]["us_per_request"]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--grids", nargs="+", default=["200x200x60", "320x320x40", "512x512x64"])
    ap.add_argument("--store", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "store_surfels": a.store, "fields": []}
    for g in [tuple(int(x) for x in s.split("x")) for s in a.grids]:
        off, on = stored_context(a.store, g), stored_context(a.store, g)
        on.field_signed_enable()
        r = {"grid": g}
        for host_copy in (True, False):
            ts = {"off": [], "on": []}
            for _ in range(a.rounds):
                for k, ctx in (("off", off), ("on", on)):
                    latency(ctx, host_copy, 3)   # warm
                    ts[k] += latency(ctx, host_copy, a.reps)
            r["host_copy" if host_copy else "resident"] = {k: spread(v) for k, v in ts.items()}
        r["kernels_signed_on"] = kernels(on, a.launches)
        off.close()
        on.close()
        res["fields"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "measure_field_signed.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
