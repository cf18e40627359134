"""Throughput of the MontgomeryPoint entry points and of the constant-time fixed-base batch on the GPU; prints one JSON
line.  Every figure is the median last_call_ms (CUDA events around the whole call, copies of host-buffer calls included)
of the timed calls, after warm-up calls of the same shape.

  mul_dev / mul_host           Scalar * MontgomeryPoint over device-resident / host buffers
  mul_bits_be_{255,512}_host   mul_bits_be over 32-byte integers read over 255 bits, and 64-byte integers over 512 bits
  to_edwards_host              MontgomeryPoint::to_edwards (random u: about half are twist points, which give None)
  mul_base_ct_{edwards,ristretto,montgomery}_host, mul_base_ct_clamped_{edwards,montgomery}_host
                               the constant-time fixed-base comb in each output form
  x25519_dev / x25519_public_keys_host   the existing X25519 ladder and public keys, measured in the same run
Only Scalar * MontgomeryPoint has a device-buffer entry point; the other calls take host buffers.

usage: python tools/bench_montgomery.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BASE = bytes([9]) + bytes(31)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def timed(fn, eng, calls, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(calls):
        fn()
        ms.append(eng.last_call_ms())
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import montgomery_oracle
    name, power = gpu_info()
    n = a.n
    rnd = os.urandom
    eng = pkg.Engine(0)
    ss = bytearray(rnd(32 * n))
    for i in range(n):
        ss[32 * i + 31] &= 0x7f                                    # Scalars: bit 255 clear
    ss = bytes(ss)
    us = rnd(32 * n)
    wide = rnd(64 * n)
    signs = rnd(n)
    d_s = torch.frombuffer(bytearray(ss), dtype=torch.uint8).cuda()
    d_u = torch.frombuffer(bytearray(us), dtype=torch.uint8).cuda()
    d_o = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    res = {"gpu": name, "power_limit": power, "n": n, "calls": a.calls}
    runs = {
        "mul_dev": lambda: eng.montgomery_mul_batch(d_s, n, d_u, n, n, device_ptrs=True, out=d_o),
        "mul_host": lambda: eng.montgomery_mul_batch(ss, n, us, n, n),
        "mul_bits_be_255_host": lambda: eng.montgomery_mul_bits_be_batch(ss, 32, n, 255, us, n, n),
        "mul_bits_be_512_host": lambda: eng.montgomery_mul_bits_be_batch(wide, 64, n, 512, us, n, n),
        "to_edwards_host": lambda: eng.montgomery_to_edwards_batch(us, signs, n),
        "mul_base_ct_edwards_host": lambda: eng.mul_base_ct_batch(ss, n, pkg.POINTS_COMPRESSED),
        "mul_base_ct_ristretto_host": lambda: eng.mul_base_ct_batch(ss, n, pkg.POINTS_RISTRETTO),
        "mul_base_ct_montgomery_host": lambda: eng.mul_base_ct_batch(ss, n, pkg.POINTS_MONTGOMERY),
        "mul_base_ct_clamped_edwards_host": lambda: eng.mul_base_ct_batch(us, n, pkg.POINTS_COMPRESSED, clamped=True),
        "mul_base_ct_clamped_montgomery_host": lambda: eng.mul_base_ct_batch(us, n, pkg.POINTS_MONTGOMERY, clamped=True),
        "x25519_dev": lambda: eng.x25519_batch(d_s, d_u, n, device_ptrs=True, out=d_o),
        "x25519_public_keys_host": lambda: eng.x25519_public_keys(us, n),
    }
    for key, fn in runs.items():
        ms = timed(fn, eng, a.calls, a.warmup)
        res[key + "_call_ms"] = ms
        res[key + "_per_s"] = n / (ms / 1e3)
    # the timed outputs against the oracle on a slice
    mo = montgomery_oracle.load()
    m = 2048
    assert eng.montgomery_mul_batch(ss[:32 * m], m, us[:32 * m], m, m) == mo.mul_bits_be_batch(ss, 32, m, 255, us, m, m)
    assert eng.montgomery_mul_bits_be_batch(wide[:64 * m], 64, m, 512, us[:32 * m], m, m) == \
        mo.mul_bits_be_batch(wide, 64, m, 512, us, m, m)
    assert eng.montgomery_to_edwards_batch(us[:32 * m], signs[:m], m)[1:] == mo.to_edwards_batch(us, signs, m)
    assert eng.mul_base_ct_batch(ss[:32 * m], m, pkg.POINTS_RISTRETTO) == mo.mul_base_batch(ss, m, montgomery_oracle.FMT_RISTRETTO)
    eng.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
