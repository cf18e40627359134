"""Per-kernel breakdown of ONE steady-state, device-resident MSM call over 2^20 extended points (the flagship
workload of bench.py), captured with torch.profiler (CUDA activities).  Run on the H100:

    python tools/profile_msm.py OUT.json [log2n] [--prep-alone]

--prep-alone profiles the construction of a VartimeEdwardsPrecomputation over the same extended points instead: the
point preparation then runs on the main stream with no sort kernels beside it (after the host-to-device copy).

Prints and writes one JSON object: the card, and every kernel / memset / memcpy of the call with its stream, start
offset from the first device activity of the call, and duration (microseconds).
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from torch.profiler import ProfilerActivity, profile
import curve25519_dalek_b200 as pkg
import bench

args = [a for a in sys.argv[1:] if not a.startswith("--")]
prep_alone = "--prep-alone" in sys.argv
out_path = args[0]
log2n = int(args[1]) if len(args) > 1 else 20
n = 1 << log2n
eng = pkg.Engine(0)
wl = bench.MsmWorkload(eng, n, n, 0, torch)


def step():
    if prep_alone:
        pkg.VartimeEdwardsPrecomputation((wl.h_points, n), engine=eng, fmt=pkg.POINTS_EXTENDED).close()
    else:
        wl.step_device_single()


for _ in range(5):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()

rows = []
for e in prof.events():
    if e.device_type != torch.autograd.DeviceType.CUDA:
        continue
    rows.append({"name": e.name, "stream": getattr(e, "device_resource_id", None),
                 "start_us": e.time_range.start, "dur_us": e.time_range.end - e.time_range.start})
rows.sort(key=lambda r: r["start_us"])
t0 = rows[0]["start_us"] if rows else 0
for r in rows:
    r["start_us"] = round(r["start_us"] - t0, 2)
    r["dur_us"] = round(r["dur_us"], 2)
by_name = {}
for r in rows:
    short = r["name"].split("(")[0].split("<")[0].replace("void ", "")
    by_name[short] = round(by_name.get(short, 0.0) + r["dur_us"], 2)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
what = ("the construction of a VartimeEdwardsPrecomputation over 2^%d extended points (bench.MsmWorkload's), after 5 "
        "warm-up constructions" if prep_alone else "one device-resident MSM call, 2^%d extended points (bench.MsmWorkload), "
        "after 5 warm-up calls") % log2n
res = {"what": what,
       "timing": "torch.profiler, CUDA activities; start_us relative to the first device activity of the call",
       "device": q,
       "span_us": round(max(r["start_us"] + r["dur_us"] for r in rows), 2) if rows else 0,
       "total_us_by_kernel": dict(sorted(by_name.items(), key=lambda kv: -kv[1])),
       "events": rows}
os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
with open(out_path, "w") as f:
    json.dump(res, f, indent=1)
print(json.dumps({k: res[k] for k in ("device", "span_us", "total_us_by_kernel")}, indent=1))
