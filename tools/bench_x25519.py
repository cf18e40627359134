"""Throughput of the X25519 entry points on the GPU and CPU baselines measured in the same run; prints one JSON line.

  dh_dev        x25519 over device-resident buffers (dalek_b200_x25519_batch_dev), median last_call_ms of the warm calls
  dh_host       the same pairs from host buffers, streamed in pieces (copies included)
  pubkeys_host  PublicKey::from over host buffers (fixed-base comb), against x25519(k, 9) through the ladder
  ladder_kernel_ms  the ladder kernel alone (last_kernel_ms of the device-resident calls)
  cpu_*         the X25519 oracle (plain C, one core) and `cryptography` (one core, and a process per host core)

usage: python tools/bench_x25519.py [--n 1048576] [--calls 21] [--warmup 3] [--out FILE]"""
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

BASE = bytes([9]) + bytes(31)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def _crypto_exchanges(args):
    from cryptography.hazmat.primitives.asymmetric.x25519 import X25519PrivateKey, X25519PublicKey
    ks, us = args
    for i in range(len(ks) // 32):
        X25519PrivateKey.from_private_bytes(ks[32 * i:32 * i + 32]).exchange(X25519PublicKey.from_public_bytes(us[32 * i:32 * i + 32]))
    return len(ks) // 32


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
    import x25519_oracle
    from cryptography.hazmat.primitives.asymmetric.x25519 import X25519PrivateKey
    name, power = gpu_info()
    n = a.n
    rnd = os.urandom
    eng = pkg.Engine(0)
    ks = rnd(32 * n)
    us = X25519PrivateKey.generate().public_key().public_bytes_raw() * n     # the ladder's cost does not depend on u
    d_k = torch.frombuffer(bytearray(ks), dtype=torch.uint8).cuda()
    d_u = torch.frombuffer(bytearray(us), dtype=torch.uint8).cuda()
    d_o = torch.empty(32 * n, dtype=torch.uint8, device="cuda")
    dev_ms, kern_ms = timed_calls(lambda: eng.x25519_batch(d_k, d_u, n, device_ptrs=True, out=d_o), eng, a.calls, a.warmup)
    host_ms, _ = timed_calls(lambda: eng.x25519_batch(ks, us, n), eng, a.calls, a.warmup)
    base_ms, _ = timed_calls(lambda: eng.x25519_batch(ks, BASE * n, n), eng, a.calls, a.warmup)
    pk_ms, _ = timed_calls(lambda: eng.x25519_public_keys(ks, n), eng, a.calls, a.warmup)
    out, _ = eng.x25519_batch(ks[:32 * 4096], us[:32 * 4096], 4096)
    xo = x25519_oracle.load()
    assert out == xo.x25519_batch(ks[:32 * 4096], us[:32 * 4096])
    assert eng.x25519_public_keys(ks[:32 * 4096], 4096) == eng.x25519_batch(ks[:32 * 4096], BASE * 4096, 4096)[0]
    # CPU baselines
    m = 4000
    t = time.perf_counter(); xo.x25519_batch(ks[:32 * m], us[:32 * m]); cpu_oracle = m / (time.perf_counter() - t)
    t = time.perf_counter(); _crypto_exchanges((ks[:32 * m], us[:32 * m])); cpu_crypto1 = m / (time.perf_counter() - t)
    cores = os.cpu_count() or 1
    per = 4000
    jobs = [(ks[32 * per * j:32 * per * (j + 1)], us[32 * per * j:32 * per * (j + 1)]) for j in range(cores)]
    with mp.get_context("spawn").Pool(cores) as pool:
        pool.map(_crypto_exchanges, jobs[:cores])          # start-up outside the timing
        t = time.perf_counter(); done = sum(pool.map(_crypto_exchanges, jobs)); cpu_cryptoN = done / (time.perf_counter() - t)
    res = {
        "gpu": name, "power_limit": power, "n": n, "calls": a.calls,
        "dh_dev_per_s": n / dev_ms * 1e3, "dh_dev_call_ms": dev_ms, "ladder_kernel_ms": kern_ms,
        "dh_host_per_s": n / host_ms * 1e3, "dh_host_call_ms": host_ms,
        "pubkeys_host_per_s": n / pk_ms * 1e3, "pubkeys_host_call_ms": pk_ms,
        "ladder_u9_host_per_s": n / base_ms * 1e3, "ladder_u9_host_call_ms": base_ms,
        "cpu_oracle_1core_per_s": cpu_oracle, "cpu_cryptography_1core_per_s": cpu_crypto1,
        "cpu_cryptography_all_cores_per_s": cpu_cryptoN, "cpu_cores": cores,
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
