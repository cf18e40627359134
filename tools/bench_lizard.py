"""Throughput of the Lizard entry points on the GPU, with CPU baselines measured in the same run; prints one JSON line and
writes it to --out (default profiles/lizard_h100.json).

Four workloads of --n items from host buffers (copies included):
  map_to_curve          32 random bytes per item
  lizard_encode         16 random bytes per item
  lizard_decode         the CompressedRistretto encodings lizard_encode gave (every item Some)
  map_to_curve_inverse  the same encodings (16 x 32 bytes and a mask out per item)
For each: the median last_call_ms of --calls warm calls (host-buffer throughput), the kernel time of one call from a
separate torch.profiler run with CUDA activities (a kernel figure), and the field multiplications per item counted from
the code (FIELD_MULS).  The GPU name, power limit and maximum SM clock are read in the same run.  CPU: the C oracle
(tests/host/lizard_oracle.c, which hashes all 16 candidates in decode, as the reference does) on one core and in 16
processes.

usage: python tools/bench_lizard.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# Field multiplications and squarings per item, counted from csrc/lizard.cuh, elligator.cuh, ge.cuh and fe64.cuh:
POW_P58 = 252 + 12            # fe_pow_p58_f64: 252 squarings, 12 multiplications (FP64)
SQRT_RATIO = 11 + POW_P58     # fe_sqrt_ratio_i<1>
RIST_MAP = 16 + SQRT_RATIO    # ristretto_elligator
RIST_COMPRESS = 14 + SQRT_RATIO
RIST_DECOMPRESS = 11 + SQRT_RATIO
JACOBI = 24 + SQRT_RATIO      # ristretto_to_jacobi: 4 squarings, 20 multiplications, one invsqrt
E_INV = 6 + SQRT_RATIO        # jacobi_e_inv_positive: a, a^2, s^2, s^4, i (s^4 - a^2), x, one invsqrt
FIELD_MULS = {
    "map_to_curve": RIST_MAP + RIST_COMPRESS,
    "lizard_encode": RIST_MAP + RIST_COMPRESS,                    # and one SHA-256 compression
    "lizard_decode": RIST_DECOMPRESS + JACOBI + 8 * E_INV,        # and eight SHA-256 compressions
    "map_to_curve_inverse": RIST_DECOMPRESS + JACOBI + 8 * E_INV,
}
KERNELS = {"map_to_curve": "k_ristretto_map_to_curve", "lizard_encode": "k_lizard_encode", "lizard_decode": "k_lizard_decode",
           "map_to_curve_inverse": "k_map_to_curve_inverse"}
CPU_PROCS = 16


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power, clock


def _cpu_job(args):
    import lizard_oracle
    kind, items = args
    o = lizard_oracle.load()
    if kind == "map_to_curve":
        o.map_to_curve_batch(items)
    elif kind == "lizard_encode":
        o.lizard_encode_batch(items)
    elif kind == "lizard_decode":
        o.lizard_decode_batch(items)
    else:
        o.map_to_curve_inverse_batch(items)
    return len(items)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "lizard_h100.json"))
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import lizard_oracle
    name, power, clock = gpu_info()
    n = a.n
    eng = pkg.Engine(0)
    raw32 = os.urandom(32 * n)
    data = os.urandom(16 * n)
    enc = eng.ristretto_lizard_encode_batch(data, n)
    calls = {
        "map_to_curve": lambda: eng.ristretto_map_to_curve_batch(raw32, n),
        "lizard_encode": lambda: eng.ristretto_lizard_encode_batch(data, n),
        "lizard_decode": lambda: eng.ristretto_lizard_decode_batch(enc, n),
        "map_to_curve_inverse": lambda: eng.ristretto_map_to_curve_inverse_batch(enc, n),
    }
    # parity of the first 4096 items with the oracle, and the full round trip, before anything is timed
    o = lizard_oracle.load()
    m = 4096
    first16 = [data[16 * i:16 * i + 16] for i in range(m)]
    first_enc = [enc[32 * i:32 * i + 32] for i in range(m)]
    assert enc[:32 * m] == b"".join(o.lizard_encode_batch(first16))
    assert eng.ristretto_map_to_curve_batch(raw32[:32 * m], m) == b"".join(o.map_to_curve_batch([raw32[32 * i:32 * i + 32] for i in range(m)]))
    rc, back, st = eng.ristretto_lizard_decode_batch(enc, n)
    assert rc == 0 and back == data
    rc, inv, masks = eng.ristretto_map_to_curve_inverse_batch(enc[:32 * m], m)
    assert (inv, masks) == o.map_to_curve_inverse_batch(first_enc)
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "n": n, "calls": a.calls, "workloads": {},
           "field_muls_note": "field multiplications + squarings per item counted from the code (SHA-256 not included); the "
                              "achieved rate is a kernel figure (kernel time from torch.profiler)"}
    for kind, fn in calls.items():
        for _ in range(a.warmup):
            fn()
        ms = []
        for _ in range(a.calls):
            fn()
            ms.append(eng.last_call_ms())
        res["workloads"][kind] = {"call_ms_median": statistics.median(ms), "call_ms_min": min(ms), "call_ms_max": max(ms),
                                  "items_per_s": n / statistics.median(ms) * 1e3, "field_muls_per_item": FIELD_MULS[kind]}
    # kernel time: a separate run under torch.profiler with CUDA activities
    from torch.profiler import profile, ProfilerActivity
    for kind, fn in calls.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                 for e in prof.key_averages() if KERNELS[kind] in e.key)
        w = res["workloads"][kind]
        w["kernel_ms"] = us / 1e3
        w["kernel_items_per_s"] = n / (us / 1e6) if us else None
        w["kernel_field_muls_G_per_s"] = (n * FIELD_MULS[kind] / (us / 1e6) / 1e9) if us else None
    # CPU: the oracle on one core, then CPU_PROCS processes
    cpu = {}
    per = 1000
    pools = {"map_to_curve": [raw32[32 * i:32 * i + 32] for i in range(per)], "lizard_encode": first16[:per],
             "lizard_decode": first_enc[:per], "map_to_curve_inverse": first_enc[:per]}
    for kind, items in pools.items():
        t = time.perf_counter(); _cpu_job((kind, items)); one = per / (time.perf_counter() - t)
        with mp.get_context("spawn").Pool(CPU_PROCS) as pool:
            pool.map(_cpu_job, [(kind, items[:10])] * CPU_PROCS)      # start-up outside the timing
            t = time.perf_counter(); done = sum(pool.map(_cpu_job, [(kind, items)] * CPU_PROCS)); alln = done / (time.perf_counter() - t)
        cpu[kind] = {"oracle_1core_per_s": one, "oracle_%d_procs_per_s" % CPU_PROCS: alln}
    res["cpu"] = dict(cpu, host_cores=os.cpu_count())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
