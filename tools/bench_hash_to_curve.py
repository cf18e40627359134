"""Throughput of the hash-to-group entry points on the GPU, with CPU baselines measured in the same run; prints one JSON
line and writes it to --out (default profiles/hash_to_curve_h100.json).

Four workloads of --n items from host buffers (copies included):
  from_uniform_bytes   64 random bytes per item
  hash_from_bytes      32-byte messages
  hash_to_curve        32-byte messages, the RFC 9380 J.5.1 DST
  encode_to_curve      32-byte messages, the RFC 9380 J.5.2 DST
For each: the median last_call_ms of --calls warm calls (host-buffer throughput), the kernel time of one call from a
separate torch.profiler run with CUDA activities (a kernel figure), and the field multiplications per item counted
from the code (FIELD_MULS) as an achieved rate beside the FP64 field rates of profiles/microbench_h100.json.  CPU: the
C oracle (tests/host/h2c_oracle.c) on one core, and one process per host core.

usage: python tools/bench_hash_to_curve.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import ctypes as C
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

DST_RO = b"QUUX-V01-CS02-with-edwards25519_XMD:SHA-512_ELL2_RO_"
DST_NU = b"QUUX-V01-CS02-with-edwards25519_XMD:SHA-512_ELL2_NU_"

# Field multiplications and squarings per item, counted from csrc/elligator.cuh, ge.cuh, fe.cuh and fe64.cuh:
POW_P58 = 252 + 12            # fe_pow_p58_f64: 252 squarings, 12 multiplications (FP64)
INVERT = 254 + 12             # fe_invert_f64 (FP64), inside ge_compress<1>
SQRT_RATIO = 11 + POW_P58     # fe_sqrt_ratio_i<1>: v^2, v^3, v^6, v^7, u v^7, r (2), check (2), -u i, r i
RIST_MAP = 16 + SQRT_RATIO    # ristretto_elligator: r, N_s, D, s', N_t, s^2, X, Z and the 4 of ge_p1p1_to_p3
GE_ADD = 9                    # ge_add: T 2d, then 8 in ge_padd
RIST_COMPRESS = 14 + SQRT_RATIO
ELL2 = 11 + POW_P58 + 13      # ell2_encode, steps 1-15, 16, 17-38
MAP = ELL2 + 7                # ell2_map_to_curve: xn, xd, tv1 and the 4 coordinates
COFACTOR = 3 * 4 + 3 + 3 + 4  # ge_mul_by_pow_2(., ., 3)
GE_COMPRESS = INVERT + 2
FIELD_MULS = {
    "from_uniform_bytes": 2 * RIST_MAP + GE_ADD + RIST_COMPRESS,
    "hash_from_bytes": 2 * RIST_MAP + GE_ADD + RIST_COMPRESS,
    "hash_to_curve": 2 * MAP + GE_ADD + COFACTOR + GE_COMPRESS,
    "encode_to_curve": MAP + COFACTOR + GE_COMPRESS,
}
KERNELS = {"from_uniform_bytes": "k_ristretto_from_uniform", "hash_from_bytes": "k_ristretto_hash_bytes",
           "hash_to_curve": "k_edwards_h2c<2>", "encode_to_curve": "k_edwards_h2c<1>"}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def _cpu_job(args):
    import h2c_oracle
    kind, items = args
    o = h2c_oracle.load()
    if kind == "from_uniform_bytes":
        o.from_uniform_batch(items)
    else:
        o.flat_batch(kind, items, DST_RO if kind == "hash_to_curve" else DST_NU)
    return len(items)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "hash_to_curve_h100.json"))
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import h2c_oracle
    name, power = gpu_info()
    n = a.n
    eng = pkg.Engine(0)
    uniform = os.urandom(64 * n)
    msgs = os.urandom(32 * n)
    offs = (C.c_uint64 * (n + 1))(*range(0, 32 * (n + 1), 32))
    calls = {
        "from_uniform_bytes": lambda: eng.ristretto_from_uniform_bytes_batch(uniform, n),
        "hash_from_bytes": lambda: eng.ristretto_hash_from_bytes_batch(msgs, offs, n),
        "hash_to_curve": lambda: eng.edwards_hash_to_curve_batch(msgs, offs, n, DST_RO),
        "encode_to_curve": lambda: eng.edwards_encode_to_curve_batch(msgs, offs, n, DST_NU),
    }
    # parity of the first 4096 items with the oracle before anything is timed
    o = h2c_oracle.load()
    m = 4096
    first = [msgs[32 * i:32 * i + 32] for i in range(m)]
    assert eng.ristretto_from_uniform_bytes_batch(uniform[:64 * m], m) == b"".join(o.from_uniform_batch([uniform[64 * i:64 * i + 64] for i in range(m)]))
    assert eng.edwards_hash_to_curve_batch(msgs[:32 * m], offs, m, DST_RO) == b"".join(o.flat_batch("hash_to_curve", first, DST_RO))
    micro = json.load(open(os.path.join(ROOT, "profiles", "microbench_h100.json")))["microbench_f64"]
    res = {"gpu": name, "power_limit": power, "n": n, "calls": a.calls, "workloads": {},
           "fp64_field_reference_G_per_s": {"f64_mul_v1_G_b2": micro.get("f64_mul_v1_G_b2"), "f64_sq_G_b2": micro.get("f64_sq_G_b2")},
           "field_muls_note": "field multiplications + squarings per item counted from the code; the achieved rate is a kernel "
                              "figure (kernel time from torch.profiler), IMAD and FP64 forms together"}
    for kind, fn in calls.items():
        for _ in range(a.warmup):
            fn()
        ms = []
        for _ in range(a.calls):
            fn()
            ms.append(eng.last_call_ms())
        res["workloads"][kind] = {"call_ms_median": statistics.median(ms), "items_per_s": n / statistics.median(ms) * 1e3,
                                  "field_muls_per_item": FIELD_MULS[kind]}
    # kernel time: a separate run under torch.profiler with CUDA activities
    from torch.profiler import profile, ProfilerActivity
    for kind, fn in calls.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tag = KERNELS[kind].split("<")[0]
        want = "Li2E" if kind == "hash_to_curve" else ("Li1E" if kind == "encode_to_curve" else "")
        us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                 for e in prof.key_averages() if tag in e.key and (not want or want in e.key or KERNELS[kind] in e.key))
        w = res["workloads"][kind]
        w["kernel_ms"] = us / 1e3
        w["kernel_items_per_s"] = n / (us / 1e6) if us else None
        w["kernel_field_muls_G_per_s"] = (n * FIELD_MULS[kind] / (us / 1e6) / 1e9) if us else None
    # CPU: the oracle on one core, then one process per core
    cpu = {}
    cores = os.cpu_count() or 1
    per = 2000
    for kind in calls:
        items = [uniform[64 * i:64 * i + 64] for i in range(per)] if kind == "from_uniform_bytes" else first[:per]
        t = time.perf_counter(); _cpu_job((kind, items)); one = per / (time.perf_counter() - t)
        with mp.get_context("spawn").Pool(cores) as pool:
            pool.map(_cpu_job, [(kind, items[:10])] * cores)            # start-up outside the timing
            t = time.perf_counter(); done = sum(pool.map(_cpu_job, [(kind, items)] * cores)); alln = done / (time.perf_counter() - t)
        cpu[kind] = {"oracle_1core_per_s": one, "oracle_all_cores_per_s": alln}
    res["cpu"] = dict(cpu, cores=cores)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
