"""Throughput of the batched Scalar arithmetic on the GPU and of the C oracle on one core; prints one JSON line and writes
it to --out (default profiles/scalar_h100.json).

Workloads (--n items, 2^20 by default; medians of --calls warm calls of last_call_ms, the device span of the call, copies
of host buffers included, and of the host wall time):
  add, mul, invert: host buffers, and device-resident (torch buffers)
  hash_from_bytes of 32-byte messages, host buffers
  Sum and Product of one segment of 16 n scalars and of n segments of 16, host buffers and device-resident
Each entry carries the work it implies per item, so that its rate can be set against the right bound: sc_mul calls (a
512-bit product and a Barrett reduction; the inversion is 253 squarings and popcount(l - 2) multiplications), SHA-512
blocks, and the bytes a device-resident call must move through HBM (inputs read once, results written once) or a host
call through PCIe.  CPU: the C oracle's scalar_add, scalar_mul and scalar_invert on one core, timed around ctypes calls
(call overhead included).  The GPU name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_scalar.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
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
L = 2**252 + 27742317777372353535851937790883648493
INVERT_MULS = 253 + bin(L - 2).count("1")          # squarings + multiplications of sc_invert
HBM_BYTES_PER_S = 3.35e12                          # H100 SXM data sheet


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
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "scalar_h100.json"))
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import oracle_lib
    name, power, clock = gpu_info()
    eng = pkg.Engine(0)
    rnd = random.Random(7)
    n = a.n
    xs = [rnd.randrange(1, L) for _ in range(2 * n)]
    flat = b"".join(x.to_bytes(32, "little") for x in xs)
    fa, fb = flat[:32 * n], flat[32 * n:]
    da = torch.frombuffer(bytearray(fa), dtype=torch.uint8).cuda()
    db = torch.frombuffer(bytearray(fb), dtype=torch.uint8).cuda()
    dout = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "n": n, "calls": a.calls, "warmup": a.warmup,
           "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S}

    def put(tag, fn, items, sc_mul_per_item, bytes_per_item, link, extra=None):
        r = timed(eng, fn, a.calls, a.warmup)
        r["items_per_s"] = items / r["call_ms"] * 1e3
        r["sc_mul_per_item"] = sc_mul_per_item
        r["bytes_per_item"] = bytes_per_item
        r["bytes_over"] = link
        r["bytes_per_s"] = r["items_per_s"] * bytes_per_item
        if sc_mul_per_item:
            r["sc_mul_per_s"] = r["items_per_s"] * sc_mul_per_item
        if link == "hbm":
            r["share_of_hbm_datasheet"] = r["bytes_per_s"] / HBM_BYTES_PER_S
        r.update(extra or {})
        res[tag] = r

    # element-wise, checked once against Python integers on a sample
    got = eng.scalar_binary_batch("mul", fa, n, fb, n, n)
    assert all(int.from_bytes(got[32 * i:32 * i + 32], "little") == xs[i] * xs[n + i] % L for i in range(0, n, 4099))
    for op, muls in (("add", 0), ("mul", 1)):
        put(op + "_host", lambda op=op: eng.scalar_binary_batch(op, fa, n, fb, n, n), n, muls, 96, "pcie")
        put(op + "_dev", lambda op=op: eng.scalar_binary_batch(op, da, n, db, n, n, device_ptrs=True, out=dout), n, muls, 96, "hbm")
    put("invert_host", lambda: eng.scalar_unary_batch("invert", fa, n), n, INVERT_MULS, 64, "pcie")
    put("invert_dev", lambda: eng.scalar_unary_batch("invert", da, n, device_ptrs=True, out=dout), n, INVERT_MULS, 64, "hbm")
    msgs = fa                                        # n messages of 32 bytes
    offs = (C.c_uint64 * (n + 1))(*range(0, 32 * n + 1, 32))
    put("hash_from_bytes_32B_host", lambda: eng.scalar_hash_from_bytes_batch(msgs, offs, n), n, 0, 64, "pcie",
        {"sha512_blocks_per_item": 1})

    # folds
    big = 16 * n
    flat_big = flat[:32 * n] * 16
    d_big = da.repeat(16)
    one = np.array([0, big], dtype=np.uint64)
    d_one = torch.from_numpy(one.view(np.int64).copy()).cuda()
    many = np.arange(0, big + 1, 16, dtype=np.uint64)
    d_many = torch.from_numpy(many.view(np.int64).copy()).cuda()
    d_fold_out = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    for op in ("sum", "product"):
        muls = 0 if op == "sum" else 1
        put("%s_1x%d_host" % (op, big), lambda op=op: eng.scalar_fold_batch(op, flat_big, one, 1), big, muls, 32, "pcie")
        put("%s_1x%d_dev" % (op, big), lambda op=op: eng.scalar_fold_batch(op, d_big, d_one, 1, device_ptrs=True, out=d_fold_out), big,
            muls, 32, "hbm")
        put("%s_%dx16_host" % (op, n), lambda op=op: eng.scalar_fold_batch(op, flat_big, many, n), big, muls, 34.5, "pcie")
        put("%s_%dx16_dev" % (op, n), lambda op=op: eng.scalar_fold_batch(op, d_big, d_many, n, device_ptrs=True, out=d_fold_out), big,
            muls, 34.5, "hbm")

    # the C oracle on one core
    orc = oracle_lib.load()
    k = 1 << 14
    o = (C.c_uint8 * 32)()
    bufs = [C.c_char_p(flat[32 * i:32 * i + 32]) for i in range(k + 1)]
    cpu = {}
    for fn, cnt in (("scalar_add", k), ("scalar_mul", k), ("scalar_invert", k // 16)):
        f = getattr(orc.lib, fn)
        t0 = time.perf_counter()
        if fn == "scalar_invert":
            for i in range(cnt):
                f(o, bufs[i])
        else:
            for i in range(cnt):
                f(o, bufs[i], bufs[i + 1])
        cpu[fn + "_per_s"] = cnt / (time.perf_counter() - t0)
    res["cpu_oracle_one_core"] = cpu
    eng.close()
    line = json.dumps(res)
    print(line)
    with open(a.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
