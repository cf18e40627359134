"""Throughput of the batched variable-time double-base scalar multiplication a_i A_i + b_i B
(dalek_b200_vartime_double_base_batch) on the GPU, with today's GPU route and the CPU oracle measured in the same run;
prints one JSON line.

  compressed_host / extended_host / ristretto_host   the three point formats from host buffers (copies included)
  compressed_dev                                     CompressedEdwardsY, device-resident buffers
  msm_batch_host / msm_batch_ristretto_host          the same work as n two-term MSMs [a_i, b_i] x [A_i, B] through
                                                     dalek_b200_msm_batch (variable time), host buffers
  cpu_oracle_1core / cpu_oracle_all_cores            tests/host/double_base_oracle.c (the reference's NAF algorithm), one
                                                     thread and one thread per core
A sample of outputs of every GPU leg is compared with the oracle.  Rates are items per second from the median
last_call_ms of the warm calls (for msm_batch the median wall time of the blocking call).

usage: python tools/bench_double_base.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import curve25519_dalek_b200 as pkg
    import double_base_oracle
    import oracle_lib
    import pyref
    name, power = gpu_info()
    n = a.n
    eng = pkg.Engine(0)
    orc = oracle_lib.load()
    dbo = double_base_oracle.load()
    rng = __import__("random").Random(1)
    ab = b"".join(rng.randrange(2**255).to_bytes(32, "little") for _ in range(2 * n))
    limbs, pts = eng.mul_base_batch(b"".join(rng.randrange(1, pyref.L).to_bytes(32, "little") for _ in range(n)), n)
    ext = bytes(limbs)
    rpts = b"".join(orc.ristretto_compress(orc.decompress(pts[32 * i:32 * i + 32])) for i in range(1024)) * (n // 1024)
    d_ab = torch.frombuffer(bytearray(ab), dtype=torch.uint8).cuda()
    d_p = torch.frombuffer(bytearray(pts), dtype=torch.uint8).cuda()
    d_o = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    res = {"gpu": name, "power_limit": power, "n": n, "calls": a.calls}

    def rate(key, fn, wall=False):
        for _ in range(a.warmup):
            fn()
        ms = []
        for _ in range(a.calls):
            t = time.perf_counter()
            fn()
            ms.append((time.perf_counter() - t) * 1e3 if wall else eng.last_call_ms())
        med = statistics.median(ms)
        res[key + "_call_ms"] = med
        res[key + "_per_s"] = n / med * 1e3

    def check(key, out, inputs, fmt):
        for i in list(range(0, n, n // 61)) + [n - 1]:
            want = dbo.one(ab[64 * i:64 * i + 32], inputs(i), ab[64 * i + 32:64 * i + 64], fmt)[0]
            assert out[32 * i:32 * i + 32] == want, (key, i)

    ed = lambda i: pts[32 * i:32 * i + 32]
    rate("compressed_host", lambda: eng.vartime_double_base_batch(ab, pts, n))
    check("compressed_host", eng.vartime_double_base_batch(ab, pts, n)[1], ed, COMPRESSED)
    rate("extended_host", lambda: eng.vartime_double_base_batch(ab, ext, n, EXTENDED))
    check("extended_host", eng.vartime_double_base_batch(ab, ext, n, EXTENDED)[1], ed, COMPRESSED)
    rate("ristretto_host", lambda: eng.vartime_double_base_batch(ab, rpts, n, RISTRETTO))
    check("ristretto_host", eng.vartime_double_base_batch(ab, rpts, n, RISTRETTO)[1], lambda i: rpts[32 * i:32 * i + 32], RISTRETTO)
    rate("compressed_dev", lambda: eng.vartime_double_base_batch(d_ab, d_p, n, device_ptrs=True, out=d_o))
    torch.cuda.synchronize()
    check("compressed_dev", bytes(d_o.cpu().numpy()), ed, COMPRESSED)
    # today's GPU route: n two-term MSMs [a_i, b_i] x [A_i, B]
    offs = np.arange(0, 2 * n + 1, 2, dtype=np.uint64)
    Bc = orc.compress(orc.basepoint())
    flat_p = b"".join(pts[32 * i:32 * i + 32] + Bc for i in range(n))
    rate("msm_batch_host", lambda: eng.msm_batch(ab, flat_p, offs, n), wall=True)
    check("msm_batch_host", eng.msm_batch(ab, flat_p, offs, n)[1], ed, COMPRESSED)
    Br = orc.ristretto_compress(orc.basepoint())
    flat_r = b"".join(rpts[32 * i:32 * i + 32] + Br for i in range(n))
    rate("msm_batch_ristretto_host", lambda: eng.msm_batch(ab, flat_r, offs, n, point_fmt=RISTRETTO), wall=True)
    res["speedup_vs_msm_batch"] = res["compressed_host_per_s"] / res["msm_batch_host_per_s"]
    res["speedup_vs_msm_batch_ristretto"] = res["ristretto_host_per_s"] / res["msm_batch_ristretto_host_per_s"]
    # CPU oracle on a slice: one thread, then one thread per core
    cores = os.cpu_count() or 1
    m1, mc = 4096, min(n, 4096 * cores)
    t = time.perf_counter(); dbo.batch(ab[:64 * m1], pts[:32 * m1], m1, COMPRESSED, 1)
    res["cpu_oracle_1core_per_s"] = m1 / (time.perf_counter() - t)
    t = time.perf_counter(); dbo.batch(ab[:64 * mc], pts[:32 * mc], mc, COMPRESSED, cores)
    res["cpu_oracle_all_cores_per_s"] = mc / (time.perf_counter() - t)
    res["cpu_cores"] = cores
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
