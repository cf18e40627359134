"""Resident verifying-key sets (ed25519_b200_key_set_*) on the GPU against ed25519_b200_verify_each_flat with default
options on the same seeded inputs, alternated call by call in the same run, outputs compared; prints one JSON line.

  w1_{set,each}_{host,dev}_k{k}     2^22 signatures (64-byte messages) under random keys of k in {256, 1024, 4096, 65536}:
                                    the set's resident tables against verify_each_flat, which de-duplicates the keys and
                                    builds their tables per call (each_comb 1: keys signing >= 8 signatures on average)
                                    or runs the plain kernel
  w2_{set,each}_n{n}                a validator set: k = 1024 keys, n in {1024, 8192, 65536} votes from host buffers (at
                                    n = 1024 every key votes once)
  w3_new_k{k}                       building a set of k in {1024, 65536} keys (copy of the keys included), then destroy
  kernels                           per-kernel device time of W1 at k = 1024 and 65536 (device buffers) and of W2, from
                                    a separate torch.profiler run
Every time is the median of the warm calls: `_ms` is the device span of the call (last_call_ms: CUDA events around the
whole call, copies included) and `_wall_ms` the host clock around the blocking call.  The card's name, power limit and
maximum SM clock are read in the same run.

usage: python tools/bench_key_set.py [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N1 = 1 << 22
W1_KS = (256, 1024, 4096, 65536)
W2_K, W2_NS = 1024, (1024, 8192, 65536)
W3_KS = (1024, 65536)
MSG = 64


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power, clock


class Workload:
    """n signatures over MSG-byte messages under random keys of k: host arrays, device copies and the inlined keys"""

    def __init__(self, eng, k, n, seed, perm=False):
        import torch
        g = np.random.Generator(np.random.PCG64(seed))
        kseeds = g.integers(0, 256, size=(k, 32), dtype=np.uint8)
        self.keys = eng.verifying_keys(kseeds, k)
        self.idx = (g.permutation(n) % k if perm else g.integers(0, k, size=n)).astype(np.uint32)
        self.offs = np.arange(n + 1, dtype=np.uint64) * MSG
        self.fl = g.integers(0, 256, size=n * MSG + 1, dtype=np.uint8)
        pks, sigs = eng.sign_batch_flat(np.ascontiguousarray(kseeds[self.idx]), self.fl, self.offs, n)
        self.pks = np.frombuffer(pks, dtype=np.uint8).copy()
        self.sg = np.frombuffer(sigs, dtype=np.uint8).copy()
        for i in g.integers(0, n, size=16):                # a few failures, so that the compared outputs are not all 0
            self.sg[64 * int(i) + 40] ^= 1
        self.n, self.k = n, k
        dev = lambda a: torch.from_numpy(a).cuda()         # noqa: E731
        self.d = [dev(self.fl), dev(self.offs.view(np.int64)), dev(self.sg), dev(self.pks), dev(self.idx.view(np.int32))]
        rc, self.h, _, _ = eng.key_set_new(self.keys, k)
        assert rc == 0

    def calls(self, eng):
        d = [t.data_ptr() for t in self.d]
        return {"set_host": lambda: eng.key_set_verify_flat(self.h, self.fl, self.offs, self.sg, self.idx, self.n),
                "each_host": lambda: eng.verify_each_flat(self.fl, self.offs, self.sg, self.pks, self.n),
                "set_dev": lambda: eng.key_set_verify_flat(self.h, d[0], d[1], d[2], d[4], self.n, device_ptrs=True),
                "each_dev": lambda: eng.verify_each_flat(d[0], d[1], d[2], d[3], self.n, device_ptrs=True)}

    def close(self, eng):
        eng.key_set_destroy(self.h)
        self.d = None


def timed(eng, fn):
    t0 = time.perf_counter()
    out = fn()
    return out, eng.last_call_ms(), (time.perf_counter() - t0) * 1e3


def alternate(eng, fns, calls, warmup):
    """name -> (median device ms, median wall ms), the calls alternated one by one; every output equal to the first's"""
    first = {}
    for _ in range(warmup):
        for name, fn in fns.items():
            first.setdefault(name, fn())
    outs = list(first.values())
    assert all(o == outs[0] for o in outs), "the set and verify_each_flat disagree"
    dev, wall = {n: [] for n in fns}, {n: [] for n in fns}
    for _ in range(calls):
        for name, fn in fns.items():
            out, ms, w = timed(eng, fn)
            assert out == outs[0]
            dev[name].append(ms); wall[name].append(w)
    return {n: (statistics.median(dev[n]), statistics.median(wall[n])) for n in fns}


def profile_kernels(out_path, calls):
    """kernel name -> device ms per call, with torch.profiler (run in a process of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import curve25519_dalek_b200 as pkg
    eng = pkg.Engine(0)
    res = {}
    cases = [("w1_k%d" % k, Workload(eng, k, N1, k), ("set_dev", "each_dev")) for k in (1024, 65536)]
    cases.append(("w2_n1024", Workload(eng, W2_K, 1024, 2, perm=True), ("set_host", "each_host")))
    for tag, w, names in cases:
        fns = w.calls(eng)
        for name in names:
            fns[name]()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    fns[name]()
                torch.cuda.synchronize()
            ker = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                if t > 0:
                    ker[e.key[:80]] = round(t / 1e3 / calls, 4)
            res["%s_%s" % (tag, name)] = ker
        w.close(eng)
    eng.close()
    with open(out_path, "w") as f:
        json.dump(res, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile-only", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.profile_only:
        profile_kernels(a.profile_only, 3)
        return
    import curve25519_dalek_b200 as pkg
    name, power, clock = gpu_info()
    eng = pkg.Engine(0)
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "calls": a.calls, "warmup": a.warmup,
           "each_comb": eng.get_option("each_comb")}
    for k in W1_KS:
        w = Workload(eng, k, N1, k)
        fns = w.calls(eng)
        for where in ("host", "dev"):
            r = alternate(eng, {c: fns[c] for c in ("set_" + where, "each_" + where)}, a.calls, a.warmup)
            for c, (ms, wall) in r.items():
                key = "w1_%s_k%d" % (c, k)
                res[key + "_ms"], res[key + "_wall_ms"] = round(ms, 3), round(wall, 3)
                res[key + "_sigs_per_s"] = round(N1 / ms * 1e3)
        w.close(eng)
    for n in W2_NS:
        w = Workload(eng, W2_K, n, n, perm=(n == W2_K))
        fns = w.calls(eng)
        r = alternate(eng, {c: fns[c] for c in ("set_host", "each_host")}, a.calls, a.warmup)
        for c, (ms, wall) in r.items():
            key = "w2_%s_n%d" % (c.split("_")[0], n)
            res[key + "_ms"], res[key + "_wall_ms"] = round(ms, 4), round(wall, 4)
        w.close(eng)
    for k in W3_KS:
        g = np.random.Generator(np.random.PCG64(k))
        keys = eng.verifying_keys(g.integers(0, 256, size=(k, 32), dtype=np.uint8), k)
        dev, wall = [], []
        for i in range(a.warmup + a.calls):
            t0 = time.perf_counter()
            rc, h, _, _ = eng.key_set_new(keys, k)
            w_ms = (time.perf_counter() - t0) * 1e3
            ms = eng.last_call_ms()
            eng.key_set_destroy(h)
            assert rc == 0
            if i >= a.warmup:
                dev.append(ms); wall.append(w_ms)
        res["w3_new_k%d_ms" % k] = round(statistics.median(dev), 3)
        res["w3_new_k%d_wall_ms" % k] = round(statistics.median(wall), 3)
    eng.close()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "kernels.json")
        subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-only", path], check=True)
        with open(path) as f:
            res["kernels"] = json.load(f)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
