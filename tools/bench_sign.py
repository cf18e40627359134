"""Throughput of the Ed25519 signer and of Ed25519ph verification on the GPU, with CPU baselines from the same run;
writes one JSON object (default profiles/sign_h100.json) and prints it.

  verifying_keys               SigningKey::from_bytes(seed).verifying_key() for n seeds
  sign_n_keys / sign_one_key   sign_flat, 32-byte messages, one key per message / one key for all
  sign_ph_ctx0 / sign_ph_ctx255  sign_prehashed with one key, empty and 255-byte context
  verify_ph_{plain,comb}[_strict]  verify_prehashed_each with all-distinct keys (plain path) and 1024 keys (comb path)
Each figure is the median device time (last_call_ms, host copies included) of --calls warm calls.  Kernel times come
from a separate torch.profiler run.  The timed outputs are checked against the C oracles on 4096 sampled indices and
must pass verify_each_flat.  CPU: `cryptography` signing on one core and on one process per available core, the oracle
on one core.

usage: python tools/bench_sign.py [--n 1048576] [--calls 21] [--warmup 3] [--out profiles/sign_h100.json]"""
import argparse
import json
import multiprocessing as mp
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _crypto_sign(args):
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    seeds, msgs = args
    for i in range(len(msgs)):
        Ed25519PrivateKey.from_private_bytes(seeds[i]).sign(msgs[i])
    return len(msgs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sign_h100.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import curve25519_dalek_b200 as pkg
    import ed25519ph_oracle
    import oracle_lib
    orc, pho = oracle_lib.load(), ed25519ph_oracle.load()
    eng = pkg.Engine(0)
    n = a.n
    gen = np.random.Generator(np.random.PCG64(2024))
    seeds = gen.integers(0, 256, size=(n, 32), dtype=np.uint8)
    msgs = gen.integers(0, 256, size=(n, 32), dtype=np.uint8)
    offs = np.arange(n + 1, dtype=np.uint64) * 32
    phs = gen.integers(0, 256, size=(n, 64), dtype=np.uint8)
    ctx255 = bytes(gen.integers(0, 256, size=255, dtype=np.uint8))
    one = seeds[0].tobytes()
    pks_all = np.frombuffer(eng.verifying_keys(seeds, n), dtype=np.uint8).reshape(n, 32)
    keys1024 = np.ascontiguousarray(pks_all[np.arange(n) % 1024])

    res, outs = {"n": n, "calls": a.calls, "message_bytes": 32}, {}

    def timed(name, fn):
        for _ in range(a.warmup):
            fn()
        ms = []
        for _ in range(a.calls):
            outs[name] = fn()
            ms.append(eng.last_call_ms())
        med = statistics.median(ms)
        res[name] = {"ms": round(med, 3), "items_per_s": round(n / med * 1e3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3)}

    timed("verifying_keys", lambda: eng.verifying_keys(seeds, n))
    timed("sign_n_keys", lambda: eng.sign_flat(seeds, n, msgs, offs, n))
    timed("sign_one_key", lambda: eng.sign_flat(one, 1, msgs, offs, n))
    timed("sign_ph_ctx0", lambda: eng.sign_prehashed(one, 1, phs, n, b"")[1])
    timed("sign_ph_ctx255", lambda: eng.sign_prehashed(one, 1, phs, n, ctx255)[1])
    rc, sig_ph_n = eng.sign_prehashed(seeds, n, phs, n, b"")
    sig_ph_1024 = np.empty((n, 64), dtype=np.uint8)
    for j in range(1024):                                                     # every 1024th item under key j
        sel = np.arange(j, n, 1024)
        sig_ph_1024[sel] = np.frombuffer(eng.sign_prehashed(seeds[j].tobytes(), 1, np.ascontiguousarray(phs[sel]), len(sel), b"")[1],
                                         dtype=np.uint8).reshape(-1, 64)
    for strict in (False, True):
        sfx = "_strict" if strict else ""
        timed("verify_ph_plain" + sfx, lambda: eng.verify_prehashed_each(phs, sig_ph_n, pks_all, n, b"", strict))
        timed("verify_ph_comb" + sfx, lambda: eng.verify_prehashed_each(phs, sig_ph_1024, keys1024, n, b"", strict))

    # outputs: oracle parity on 4096 sampled indices, and every signature verifies
    rnd = random.Random(1)
    idx = sorted(rnd.sample(range(n), 4096))
    pk_b = outs["verifying_keys"]
    sn, s1 = outs["sign_n_keys"], outs["sign_one_key"]
    p0, p255 = outs["sign_ph_ctx0"], outs["sign_ph_ctx255"]
    pk1 = orc.public_key(one)
    for i in idx:
        s, m, ph = seeds[i].tobytes(), msgs[i].tobytes(), phs[i].tobytes()
        assert pk_b[32 * i:32 * i + 32] == orc.public_key(s)
        assert sn[64 * i:64 * i + 64] == orc.sign(m, s)
        assert s1[64 * i:64 * i + 64] == orc.sign(m, one)
        assert p0[64 * i:64 * i + 64] == pho.sign_prehashed(one, ph, b"")[1]
        assert p255[64 * i:64 * i + 64] == pho.sign_prehashed(one, ph, ctx255)[1]
    for sigs, keys in ((sn, pks_all), (s1, np.tile(np.frombuffer(pk1, dtype=np.uint8), (n, 1)))):
        for strict in (False, True):
            assert eng.verify_each_flat(msgs, offs, sigs, np.ascontiguousarray(keys), n, strict=strict)[0] == 0
    for name in ("verify_ph_plain", "verify_ph_comb", "verify_ph_plain_strict", "verify_ph_comb_strict"):
        assert outs[name][0] == 0
    res["outputs_checked"] = {"oracle_sampled_indices": len(idx), "verify_each_all": True}

    # kernel times: a separate profiled run, one profiler session per call so that each call's kernels stay apart
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    calls = {"sign_n_keys": lambda: eng.sign_flat(seeds, n, msgs, offs, n),
             "sign_one_key": lambda: eng.sign_flat(one, 1, msgs, offs, n),
             "sign_ph_ctx255": lambda: eng.sign_prehashed(one, 1, phs, n, ctx255),
             "verify_ph_plain": lambda: eng.verify_prehashed_each(phs, sig_ph_n, pks_all, n, b"", False),
             "verify_ph_comb": lambda: eng.verify_prehashed_each(phs, sig_ph_1024, keys1024, n, b"", False)}
    kern = {}
    for name, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        kern[name] = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and "k_" in ev.key:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                kern[name][ev.key.split("(")[0][:60]] = {"total_ms": round(t / 1e3, 3), "count": ev.count}
        kern[name]["kernels_ms"] = round(sum(v["total_ms"] for v in kern[name].values()), 3)
    res["kernels_profiled"] = kern

    # CPU baselines
    m = 20000
    t0 = time.perf_counter()
    _crypto_sign(([seeds[i].tobytes() for i in range(m)], [msgs[i].tobytes() for i in range(m)]))
    res["cpu_cryptography_1core_per_s"] = round(m / (time.perf_counter() - t0))
    procs = len(os.sched_getaffinity(0))
    chunks = [([seeds[i].tobytes() for i in range(k, 16 * m, procs)], [msgs[i].tobytes() for i in range(k, 16 * m, procs)])
              for k in range(procs)]
    with mp.Pool(procs) as pool:
        pool.map(_crypto_sign, [([c[0][0]], [c[1][0]]) for c in chunks])
        t0 = time.perf_counter()
        done = sum(pool.map(_crypto_sign, chunks))
        res["cpu_cryptography_procs_per_s"] = round(done / (time.perf_counter() - t0))
    res["cpu_procs"] = procs
    m = 5000
    t0 = time.perf_counter()
    for i in range(m):
        orc.sign(msgs[i].tobytes(), seeds[i].tobytes())
    res["cpu_oracle_1core_per_s"] = round(m / (time.perf_counter() - t0))
    res.update(gpu_info())
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
