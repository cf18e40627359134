"""Throughput of ed25519_b200_verify_each_flat from pinned host buffers on the plain path (option each_comb = 0): 2^22
signatures by distinct keys, streamed in pieces over two streams (copies included).  bench.py times verify_each with
1024 keys (the per-key comb path) and from device buffers; this is the path a batch of one-off keys takes from host memory.
Prints one JSON line.

usage: python tools/bench_verify_each_host.py [--n 4194304] [--calls 11] [--warmup 2] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 22)
    ap.add_argument("--calls", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import curve25519_dalek_b200 as pkg
    name, power = gpu_info()
    n = a.n
    eng = pkg.Engine(0)
    eng.set_option("each_comb", 0)
    flat, offs, sigs, pks = bench.build_verify_inputs(eng, n, nkeys=n)
    h = [torch.from_numpy(x if x.dtype == np.uint8 else x.view(np.int64)).pin_memory() for x in (flat, offs, sigs, pks)]
    res = np.zeros(n, dtype=np.uint8)

    def call():
        rc = eng.lib.ed25519_b200_verify_each_flat(eng.h, h[0].data_ptr(), h[1].data_ptr(), h[2].data_ptr(), h[3].data_ptr(), n, 0,
                                                   res.ctypes.data)
        if rc != 0:
            raise SystemExit("verify_each rejected valid signatures (rc=%d)" % rc)

    for _ in range(a.warmup):
        call()
    wall, span = [], []
    for _ in range(a.calls):
        t = time.perf_counter()
        call()
        wall.append((time.perf_counter() - t) * 1e3)
        span.append(eng.last_kernel_ms()[0])
    out = {"gpu": name, "power_limit": power, "n": n, "calls": a.calls, "path": "plain kernel, pinned host buffers, distinct keys",
           "sigs_per_s": n / statistics.median(wall) * 1e3, "call_ms_median": statistics.median(wall),
           "call_ms_min": min(wall), "call_ms_max": max(wall), "device_span_ms_median": statistics.median(span),
           "launches_per_call": eng.last_kernel_ms()[1]}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
