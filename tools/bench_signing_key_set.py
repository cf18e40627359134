"""Resident signing-key sets (ed25519_b200_signing_key_set_*) and hazmat signing (ed25519_b200_raw_sign_flat) on the GPU
against ed25519_b200_sign_flat on the same seeded inputs, alternated call by call in the same run, outputs compared;
prints one JSON line.

  w1_k{k}_{name}     2^20 32-byte messages from host buffers, each signed under a random key of k in {1, 1024, 65536,
                     2^20}:
                       set_host    the set, messages and indices from host buffers
                       set_dev     the set, every buffer in device memory (the device-resident rate)
                       sign_seeds  sign_flat with one seed per message (the key derived again for every message)
                       raw_sign    raw_sign_flat with one expanded key (SHA-512 of the seed) and verifying key per message
                     All four give the same bytes.  At k = 1 the group also runs sign_one_seed: sign_flat with one seed
                     for the whole batch, which derives the key once per call.
  w3_new_k{k}        building a set of k in {1024, 65536, 2^20} keys from seeds (copy of the seeds included), then destroy
  oracle_checked     signatures of sampled messages checked against the C oracle
Every time is the median of the warm calls: `_ms` is the device span of the call (last_call_ms: CUDA events around the
whole call, copies included) and `_wall_ms` the host clock around the blocking call.  The card's name, power limit and
maximum SM clock are read in the same run.

usage: python tools/bench_signing_key_set.py [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N = 1 << 20
W1_KS = (1, 1024, 65536, 1 << 20)
W3_KS = (1024, 65536, 1 << 20)
MSG = 32


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power, clock


def timed(eng, fn):
    t0 = time.perf_counter()
    out = fn()
    return out, eng.last_call_ms(), (time.perf_counter() - t0) * 1e3


def alternate(eng, fns, calls, warmup):
    """name -> (median device ms, median wall ms), the calls alternated one by one"""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    dev, wall = {n: [] for n in fns}, {n: [] for n in fns}
    for _ in range(calls):
        for name, fn in fns.items():
            _, ms, w = timed(eng, fn)
            dev[name].append(ms); wall[name].append(w)
    return {n: (statistics.median(dev[n]), statistics.median(wall[n])) for n in fns}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    from curve25519_dalek_b200.engine import SIGNING_KEY_SEED
    import oracle_lib
    orc = oracle_lib.load()
    eng = pkg.Engine(0)
    name, power, clock = gpu_info()
    out = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "n": N, "msg_bytes": MSG, "calls": a.calls,
           "warmup": a.warmup}
    g = np.random.Generator(np.random.PCG64(2026))
    offs = np.arange(N + 1, dtype=np.uint64) * MSG
    fl = g.integers(0, 256, size=N * MSG + 1, dtype=np.uint8)
    d_fl, d_offs = torch.from_numpy(fl).cuda(), torch.from_numpy(offs.view(np.int64)).cuda()
    d_out = torch.empty(64 * N, dtype=torch.uint8, device="cuda")
    checked = 0
    for k in W1_KS:
        seeds = g.integers(0, 256, size=(k, 32), dtype=np.uint8)
        idx = g.integers(0, k, size=N).astype(np.uint32)
        per_msg = np.ascontiguousarray(seeds[idx])
        esks = np.frombuffer(b"".join(hashlib.sha512(s.tobytes()).digest() for s in seeds), dtype=np.uint8).reshape(k, 64)
        rc, h, _ = eng.signing_key_set_new(seeds, k, SIGNING_KEY_SEED)
        assert rc == 0
        vks = np.frombuffer(eng.signing_key_set_verifying_keys(h), dtype=np.uint8).reshape(k, 32)
        esk_msg, vk_msg = np.ascontiguousarray(esks[idx]), np.ascontiguousarray(vks[idx])
        d_idx = torch.from_numpy(idx.view(np.int32)).cuda()
        fns = {"set_host": lambda: eng.signing_key_set_sign_flat(h, fl, offs, idx, N),
               "set_dev": lambda: eng.signing_key_set_sign_flat(h, d_fl.data_ptr(), d_offs.data_ptr(), d_idx.data_ptr(), N,
                                                                device_ptrs=True, out=d_out.data_ptr()),
               "sign_seeds": lambda: eng.sign_flat(per_msg, N, fl, offs, N),
               "raw_sign": lambda: eng.raw_sign_flat(esk_msg, vk_msg, N, fl, offs, N)}
        if k == 1:
            fns["sign_one_seed"] = lambda: eng.sign_flat(seeds[0].tobytes(), 1, fl, offs, N)
        want = fns["set_host"]()
        fns["set_dev"]()
        assert d_out.cpu().numpy().tobytes() == want, "set_dev differs from set_host at k = %d" % k
        for nm in ("sign_seeds", "raw_sign") + (("sign_one_seed",) if k == 1 else ()):
            assert fns[nm]() == want, "%s differs from set_host at k = %d" % (nm, k)
        for i in g.integers(0, N, size=32):
            i = int(i)
            assert want[64 * i:64 * i + 64] == orc.sign(fl[MSG * i:MSG * i + MSG].tobytes(), seeds[idx[i]].tobytes()), i
            checked += 1
        for nm, (ms, wall) in alternate(eng, fns, a.calls, a.warmup).items():
            out["w1_k%d_%s_ms" % (k, nm)] = round(ms, 3)
            out["w1_k%d_%s_wall_ms" % (k, nm)] = round(wall, 3)
            out["w1_k%d_%s_Msigs_per_s" % (k, nm)] = round(N / ms / 1e3, 2)
        eng.signing_key_set_destroy(h)
        del per_msg, esk_msg, vk_msg, d_idx
    for k in W3_KS:
        seeds = g.integers(0, 256, size=(k, 32), dtype=np.uint8)
        dev, wall = [], []
        for j in range(a.warmup + a.calls):
            t0 = time.perf_counter()
            rc, h, _ = eng.signing_key_set_new(seeds, k, SIGNING_KEY_SEED)
            w = (time.perf_counter() - t0) * 1e3
            assert rc == 0
            ms = eng.last_call_ms()
            eng.signing_key_set_destroy(h)
            if j >= a.warmup:
                dev.append(ms); wall.append(w)
        out["w3_new_k%d_ms" % k] = round(statistics.median(dev), 3)
        out["w3_new_k%d_wall_ms" % k] = round(statistics.median(wall), 3)
    out["oracle_checked"] = checked
    eng.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
