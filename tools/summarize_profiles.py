"""Turns the scratch ncu outputs of tools/gpu_prof.sh (gpurun_out/<tag>/) into the small tracked summaries under profiles/:
  <name>_launches.csv            the raw launch list (every launch of tools/prof_step.py 32 3, gpu__time_duration)
  <name>_launches_summary.csv    per kernel: launches, total / average time, share of the step
  <name>_ncu_digest.csv          one --set full launch of each kernel: time, instructions, issue / occupancy, pipes, DRAM bytes, top stalls
  traffic.json                   DRAM read + write bytes per 32-frame step, per kernel and per bench.py phase (roofline.traffic)
usage: python tools/summarize_profiles.py <name> gpurun_out/<tag>"""
import collections
import csv
import json
import os
import subprocess
import sys

name, src = sys.argv[1], sys.argv[2]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
out = os.path.join(ROOT, "profiles")
os.makedirs(out, exist_ok=True)
BENCH = {"k_seed_init": "seed_init", "k_assign2<1>": "slic_assign_first", "k_assign2<0>": "slic_assign", "k_gather": "slic_gather",
         "k_newton_hard": "slic_newton", "k_plane_gather": "plane_gather", "k_gn_solve": "plane_solve",
         "k_fuse": "surfel_fuse", "k_init_surfels": "surfel_init", "k_repack": "repack"}
PER_STEP = {"k_seed_init": 1, "k_assign2<1>": 1, "k_assign2<0>": 2, "k_gather": 3, "k_newton_hard": 3, "k_plane_gather": 1,
            "k_gn_solve": 1, "k_fuse": 1, "k_init_surfels": 1}
PHASE = {"slic_assign_first": "slic_assign"}


def short(kn):
    kn = kn.replace("void ", "").split("(DsmDev")[0].split("(const")[0]
    return kn.replace("(bool)", "").strip()


# ---- launch list
launches = os.path.join(src, "launches.csv")
rows = [r for r in csv.reader(open(launches)) if len(r) > 5 and r[0].isdigit()]
agg = collections.OrderedDict()
for r in rows:
    a = agg.setdefault(short(r[4]), [0, 0.0])
    a[0] += 1
    a[1] += float(r[-1].replace(",", ""))
tot = sum(v[1] for v in agg.values())
with open(os.path.join(out, f"{name}_launches_summary.csv"), "w") as f:
    w = csv.writer(f)
    w.writerow(["kernel", "bench_name", "launches", "total_us", "avg_us", "share_pct"])
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        w.writerow([k, BENCH.get(k, k), v[0], f"{v[1] / 1e3:.1f}", f"{v[1] / v[0] / 1e3:.2f}", f"{v[1] / tot * 100:.1f}"])
subprocess.run(["cp", launches, os.path.join(out, f"{name}_launches.csv")])

# ---- full set
rep = os.path.join(src, "full.ncu-rep")
dig = os.path.join(out, f"{name}_ncu_digest.csv")
subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_digest.py"), rep, dig], check=True)
seen, keep = set(), []
rows = list(csv.DictReader(open(dig)))
for r in rows:
    k = short(r["kernel"])
    r["kernel"] = k
    if k not in seen:
        seen.add(k)
        keep.append(r)
with open(dig, "w") as f:
    w = csv.DictWriter(f, fieldnames=list(keep[0].keys()))
    w.writeheader()
    w.writerows(keep)
traffic, phases = {}, {}
for r in keep:
    k = r["kernel"]
    mb = float(r["dramRdMB"]) + float(r["dramWrMB"])
    traffic[k] = {"dram_bytes_per_launch": mb * 1e6, "launches_per_step": PER_STEP.get(k, 0)}
    ph = PHASE.get(BENCH.get(k, k), BENCH.get(k, k))
    phases[ph] = phases.get(ph, 0.0) + mb * 1e6 * PER_STEP.get(k, 0)
json.dump({"source": f"{name}: ncu --set full --clock-control none, tools/prof_step.py 32 3 (32-frame resident batch), one launch of each kernel",
           "kernels": traffic, **{k: v for k, v in phases.items()}, "step_total": sum(phases.values())},
          open(os.path.join(out, "traffic.json"), "w"), indent=1)
print("wrote", dig, "and traffic.json; step DRAM bytes:", sum(phases.values()) / 1e6, "MB")
