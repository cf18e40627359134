"""Throughput of variable-base scalar multiplication (dalek_b200_mul_batch) and the torsion check on the GPU, with the
in-tree and CPU comparisons measured in the same run; prints one JSON line.

  edwards_dev / edwards_host   s_i * P_i, CompressedEdwardsY, device-resident and host buffers (copies included)
  edwards_extended_dev         the same from extended limbs (no square root of decompression: the kernel's work closest
                               to k_ct_scalar_mul's, which starts from prepared points and does not encode)
  ristretto_host               s_i * P_i, CompressedRistretto, host buffers
  shared_scalar_host           one scalar, n points
  shared_point_*               one point, n scalars: the path the call chooses (comb from VARMUL_COMB_MIN items) against the
                               per-item path forced by repeating the point, at sizes either side of the cutoff
  torsion_host                 is_small_order / is_torsion_free flags
  ct_scalar_mul_kernel_ms      k_ct_scalar_mul (the products of dalek_b200_edwards_ct_msm, its last_kernel_ms) at the same n
  x25519_dev                   the X25519 ladder from device buffers (about the same number of field operations)
  cpu_oracle_*                 the C oracle's ge_scalarmul + compress, one core and a thread per core
Rates are items per second from the median last_call_ms of the warm calls.

usage: python tools/bench_scalar_mul.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import concurrent.futures
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COMPRESSED, RISTRETTO = 0, 2
COMB_MIN = 16384                   # varmul.cu VARMUL_COMB_MIN


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def timed_calls(fn, eng, calls, warmup):
    for _ in range(warmup):
        fn()
    call, kern = [], []
    for _ in range(calls):
        fn()
        call.append(eng.last_call_ms())
        kern.append(eng.last_kernel_ms()[0])
    return statistics.median(call), statistics.median(kern)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import oracle_lib
    import pyref
    name, power = gpu_info()
    n = a.n
    eng = pkg.Engine(0)
    orc = oracle_lib.load()
    rng = __import__("random").Random(1)
    ss = b"".join(rng.randrange(pyref.L).to_bytes(32, "little") for _ in range(n))
    _, pts = eng.mul_base_batch(b"".join(rng.randrange(pyref.L).to_bytes(32, "little") for _ in range(n)), n)
    rpts = b"".join(orc.ristretto_compress(orc.decompress(pts[32 * i:32 * i + 32])) for i in range(1024)) * (n // 1024)
    d_s = torch.frombuffer(bytearray(ss), dtype=torch.uint8).cuda()
    d_p = torch.frombuffer(bytearray(pts), dtype=torch.uint8).cuda()
    d_o = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    res = {"gpu": name, "power_limit": power, "n": n, "calls": a.calls}

    def rate(key, fn, m=n):
        ms, kern = timed_calls(fn, eng, a.calls, a.warmup)
        res[key + "_per_s"] = m / ms * 1e3
        res[key + "_call_ms"] = ms
        return ms, kern

    _, k = rate("edwards_dev", lambda: eng.mul_batch(d_s, n, d_p, n, n, device_ptrs=True, out=d_o))
    res["edwards_dev_kernel_ms"] = k
    limbs, _ = eng.mul_base_batch(ss[:32 * 1024], 1024, want_compressed=False)
    d_x = torch.frombuffer(bytearray(bytes(limbs) * (n // 1024)), dtype=torch.uint8).cuda()
    _, k = rate("edwards_extended_dev", lambda: eng.mul_batch(d_s, n, d_x, n, n, pkg.POINTS_EXTENDED, device_ptrs=True, out=d_o))
    res["edwards_extended_dev_kernel_ms"] = k
    rate("edwards_host", lambda: eng.mul_batch(ss, n, pts, n, n))
    rate("ristretto_host", lambda: eng.mul_batch(ss, n, rpts, n, n, RISTRETTO))
    rate("shared_scalar_host", lambda: eng.mul_batch(ss[:32], 1, pts, n, n))
    P = pts[:32]
    for m in (COMB_MIN // 4, COMB_MIN - 1, COMB_MIN, 4 * COMB_MIN, n):
        rate("shared_point_%d" % m, lambda: eng.mul_batch(ss, m, P, 1, m), m)
        rate("shared_point_per_item_%d" % m, lambda: eng.mul_batch(ss, m, P * m, m, m), m)
    rate("torsion_host", lambda: eng.torsion_batch(pts, n))
    _, k = timed_calls(lambda: eng.edwards_ct_msm(ss, pts, n), eng, a.calls, a.warmup)
    res["ct_scalar_mul_kernel_ms"] = k
    res["ct_scalar_mul_kernel_per_s"] = n / k * 1e3
    d_u = torch.frombuffer(bytearray((bytes([9]) + bytes(31)) * n), dtype=torch.uint8).cuda()
    _, k = rate("x25519_dev", lambda: eng.x25519_batch(d_s, d_u, n, device_ptrs=True, out=d_o))
    # outputs against the oracle on a sample, both shared-point paths included
    m = 2048
    out = eng.mul_batch(ss[:32 * m], m, pts[:32 * m], m, m)[1]
    for i in range(0, m, 97):
        s = ss[32 * i:32 * i + 32]
        assert out[32 * i:32 * i + 32] == orc.compress(orc.scalarmul(s, orc.decompress(pts[32 * i:32 * i + 32])))
    assert eng.mul_batch(ss, COMB_MIN, P, 1, COMB_MIN)[1] == eng.mul_batch(ss, COMB_MIN, P * COMB_MIN, COMB_MIN, COMB_MIN)[1]
    # CPU oracle: one core, then one thread per core (ctypes releases the GIL during the call)
    pts_o = [orc.decompress(pts[32 * i:32 * i + 32]) for i in range(512)]
    scal = [ss[32 * i:32 * i + 32] for i in range(512)]

    def cpu_chunk(_):
        for s, p in zip(scal, pts_o):
            orc.compress(orc.scalarmul(s, p))
        return len(scal)
    t = time.perf_counter(); cpu_chunk(0); res["cpu_oracle_1core_per_s"] = len(scal) / (time.perf_counter() - t)
    cores = os.cpu_count() or 1
    with concurrent.futures.ThreadPoolExecutor(cores) as ex:
        t = time.perf_counter(); done = sum(ex.map(cpu_chunk, range(2 * cores)))
        res["cpu_oracle_all_cores_per_s"] = done / (time.perf_counter() - t)
    res["cpu_cores"] = cores
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
