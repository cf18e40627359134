"""Throughput of the batched group operations on the GPU against the same work through msm_batch with unit scalars and
against the C oracle on one core; prints one JSON line and writes it to --out (default profiles/point_ops_h100.json).

Workloads (--n items, 2^20 by default; medians of --calls warm calls of last_call_ms, the device span of the call, copies
of host buffers included, and of the host wall time):
  add / sub, Edwards and Ristretto, compressed in and out, host buffers
  add, EXTENDED in and out, device buffers
  sum of one segment of 16 n points: compressed from host buffers, and EXTENDED on the device
  sum of n / 16 segments of 16 compressed points, host buffers
  the three sums again through msm_batch (variable time) with every scalar 1
The points are n multiples of the basepoint; the 16 n-point segment repeats them 16 times (decoding costs the same).
CPU: the C oracle's decompression and addition, one core, timed around C loops (ctypes call overhead included for the
decompression).  The GPU name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_point_ops.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return [s.strip() for s in r.stdout.splitlines()[0].split(",")]


def timed(eng, fn, calls, warmup):
    import torch
    for _ in range(warmup):
        fn()
    dev, host = [], []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(eng.last_call_ms())
    return {"call_ms": statistics.median(dev), "host_ms": statistics.median(host)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "point_ops_h100.json"))
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import oracle_lib
    name, power, clock = gpu_info()
    eng = pkg.Engine(0)
    rnd = random.Random(7)
    n = a.n
    CMP, EXT, RIS = pkg.POINTS_COMPRESSED, pkg.POINTS_EXTENDED, pkg.POINTS_RISTRETTO
    sc = b"".join(rnd.randrange(1, 2**252).to_bytes(32, "little") for _ in range(2 * n))
    limbs, comp = eng.mul_base_batch(sc, 2 * n)
    limbs = bytes(limbs)
    ea, eb = comp[:32 * n], comp[32 * n:]
    ra, rb = (eng.mul_base_ct_batch(sc[:32 * n], n, RIS), eng.mul_base_ct_batch(sc[32 * n:], n, RIS))
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "n": n, "calls": a.calls, "warmup": a.warmup}

    def add(tag, x, y, fmt, sub):
        res[tag] = timed(eng, lambda: eng.point_add_batch(x, n, y, n, n, fmt, sub=sub), a.calls, a.warmup)
        res[tag]["items_per_s"] = n / res[tag]["call_ms"] * 1e3

    add("edwards_add_host", ea, eb, CMP, False)
    add("edwards_sub_host", ea, eb, CMP, True)
    add("ristretto_add_host", ra, rb, RIS, False)
    add("ristretto_sub_host", ra, rb, RIS, True)
    d_la = torch.frombuffer(bytearray(limbs[:160 * n]), dtype=torch.uint8).cuda()
    d_lb = torch.frombuffer(bytearray(limbs[160 * n:]), dtype=torch.uint8).cuda()
    d_out = torch.empty(160 * n, dtype=torch.uint8, device="cuda")
    res["edwards_add_extended_dev"] = timed(eng, lambda: eng.point_add_batch(d_la, n, d_lb, n, n, EXT, out_fmt=EXT, device_ptrs=True,
                                                                             out=d_out), a.calls, a.warmup)
    res["edwards_add_extended_dev"]["items_per_s"] = n / res["edwards_add_extended_dev"]["call_ms"] * 1e3

    # sums and the same sums through msm_batch with unit scalars
    big = 16 * n
    big_comp = ea * 16
    one_off = np.array([0, big], dtype=np.uint64)
    d_big = d_la.repeat(16)
    d_one_off = torch.from_numpy(one_off.view(np.int64).copy()).cuda()
    d_out_big = torch.empty(160, dtype=torch.uint8, device="cuda")
    small_m = n // 16
    small_off = np.arange(0, n + 1, 16, dtype=np.uint64)
    ones = (1).to_bytes(32, "little")
    d_ones = torch.frombuffer(bytearray(ones * big), dtype=torch.uint8).cuda()
    shapes = {
        "sum_1x%d_compressed_host" % big: (lambda: eng.point_sum_batch(big_comp, one_off, 1, CMP),
                                           lambda: eng.msm_batch(ones * big, big_comp, one_off, 1, CMP), big),
        "sum_1x%d_extended_dev" % big: (lambda: eng.point_sum_batch(d_big, d_one_off, 1, EXT, out_fmt=EXT, device_ptrs=True, out=d_out_big),
                                        lambda: eng.msm_batch(d_ones, d_big, d_one_off, 1, EXT, device_ptrs=True), big),
        "sum_%dx16_compressed_host" % small_m: (lambda: eng.point_sum_batch(ea, small_off, small_m, CMP),
                                                lambda: eng.msm_batch(ones * n, ea, small_off, small_m, CMP), n),
    }
    for tag, (fs, fm, pts) in shapes.items():
        if not tag.endswith("_dev"):
            assert fs()[1] == fm()[1], tag
        res[tag] = timed(eng, fs, a.calls, a.warmup)
        res[tag]["points_per_s"] = pts / res[tag]["call_ms"] * 1e3
        res[tag + "_msm_batch_unit"] = timed(eng, fm, a.calls, a.warmup)
        res[tag + "_msm_batch_unit"]["points_per_s"] = pts / res[tag + "_msm_batch_unit"]["call_ms"] * 1e3
        res[tag]["speedup_vs_msm_batch"] = res[tag + "_msm_batch_unit"]["call_ms"] / res[tag]["call_ms"]

    # the C oracle on one core
    orc = oracle_lib.load()
    k = 1 << 14
    P = (oracle_lib.P3 * k)()
    t0 = time.perf_counter()
    for i in range(k):
        orc.lib.ge_decompress(C.byref(P[i]), C.c_char_p(ea[32 * i:32 * i + 32]))
    dec_s = time.perf_counter() - t0
    out = (C.c_uint8 * 32)()
    orc.lib.oracle_sum_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    t0 = time.perf_counter()
    orc.lib.oracle_sum_points(out, None, P, k)
    add_s = time.perf_counter() - t0
    res["cpu_oracle_one_core"] = {"decompress_per_s": k / dec_s, "add_per_s": k / add_s}
    eng.close()
    line = json.dumps(res)
    print(line)
    with open(a.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
