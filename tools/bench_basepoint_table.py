"""Resident basepoint tables (dalek_b200_basepoint_tables_*) on the GPU, each measurement beside what a user has without
them, alternated call by call in the same run; prints one JSON line.

  new_k{1,1024,65536}                   building k tables (copy of the points included), then destroy
  one_table_{host,dev}_{n}              s_i P from one resident table, n in {256, 4096, 16384, 2^20}
  broadcast_{host,dev}_{n}              mul_batch with the point broadcast (comb from VARMUL_COMB_MIN items, a table built
                                        per call; per item below it), same scalars
  many_tables_{host,dev}_k{k}           2^20 items with random indices into k tables, k in {64, 4096, 65536}, grouped by
                                        table on the device first (option "bpt_group" 1, the default)
  ungrouped_{host,dev}_k{k}             the same with every lane reading its own table (option "bpt_group" 0)
  per_item_{host,dev}_k{k}              mul_batch with the point P_{t_i} per item, same scalars and points
  kernels                               per-kernel device time of the same calls, from a separate torch.profiler run
Every time is the median of the warm calls' device span (last_call_ms: CUDA events around the whole call, copies
included).  The card's name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_basepoint_table.py [--calls 21] [--warmup 3] [--out FILE]"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

L = 2**252 + 27742317777372353535851937790883648493
N_BIG = 1 << 20
ONE_SIZES = (256, 4096, 16384, N_BIG)
NEW_KS = (1, 1024, 65536)
MANY_KS = (64, 4096, 65536)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power, clock


class Inputs:
    def __init__(self, eng):
        import torch
        rnd = random.Random(1)
        self.ss = b"".join(rnd.randrange(L).to_bytes(32, "little") for _ in range(N_BIG))
        kmax = max(MANY_KS + NEW_KS)
        _, self.pts = eng.mul_base_batch(b"".join(rnd.randrange(1, L).to_bytes(32, "little") for _ in range(kmax)), kmax)
        self.idx = {k: [rnd.randrange(k) for _ in range(N_BIG)] for k in MANY_KS}
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()   # noqa: E731
        self.d_s = dev(self.ss)
        self.d_o = torch.empty(32 * N_BIG, dtype=torch.uint8, device="cuda")
        import array
        self.idx_b = {k: array.array("I", v).tobytes() for k, v in self.idx.items()}
        self.d_idx = {k: dev(v) for k, v in self.idx_b.items()}
        # mul_batch's inputs with the point of each item's table
        self.per_item = {k: b"".join(self.pts[32 * t:32 * t + 32] for t in v) for k, v in self.idx.items()}
        self.d_per_item = {k: dev(v) for k, v in self.per_item.items()}
        self.d_p0 = dev(self.pts[:32])


def configs(eng, x, handles):
    """name -> zero-argument call, in the order they are measured; each group of groups() shares its inputs"""
    h1 = handles[1]
    c = {}

    def grouped(v, fn):
        def call():
            eng.set_option("bpt_group", v)
            return fn()
        return call
    for n in ONE_SIZES:
        ss = x.ss[:32 * n]
        c["one_table_host_%d" % n] = lambda ss=ss, n=n: eng.basepoint_tables_mul(h1, ss, None, n)
        c["broadcast_host_%d" % n] = lambda ss=ss, n=n: eng.mul_batch(ss, n, x.pts[:32], 1, n)
        c["one_table_dev_%d" % n] = lambda n=n: eng.basepoint_tables_mul(h1, x.d_s, None, n, device_ptrs=True, out=x.d_o)
        c["broadcast_dev_%d" % n] = lambda n=n: eng.mul_batch(x.d_s, n, x.d_p0, 1, n, device_ptrs=True, out=x.d_o)
    for k in MANY_KS:
        hk = handles[k]
        host = lambda hk=hk, k=k: eng.basepoint_tables_mul(hk, x.ss, x.idx_b[k], N_BIG)                      # noqa: E731
        dev = lambda hk=hk, k=k: eng.basepoint_tables_mul(hk, x.d_s, x.d_idx[k], N_BIG, device_ptrs=True, out=x.d_o)  # noqa: E731
        c["many_tables_host_k%d" % k] = grouped(1, host)
        c["ungrouped_host_k%d" % k] = grouped(0, host)
        c["per_item_host_k%d" % k] = lambda k=k: eng.mul_batch(x.ss, N_BIG, x.per_item[k], N_BIG, N_BIG)
        c["many_tables_dev_k%d" % k] = grouped(1, dev)
        c["ungrouped_dev_k%d" % k] = grouped(0, dev)
        c["per_item_dev_k%d" % k] = lambda k=k: eng.mul_batch(x.d_s, N_BIG, x.d_per_item[k], N_BIG, N_BIG, device_ptrs=True,
                                                              out=x.d_o)
    eng.set_option("bpt_group", 1)
    return c


def groups(names):
    """the measured names in groups alternated call by call: the one-table pairs, the many-table triples"""
    out, i = [], 0
    while i < len(names):
        w = 2 if names[i].startswith("one_table") else 3
        out.append(names[i:i + w])
        i += w
    return out


def check_outputs(eng, x, handles):
    """the tables give mul_batch's bytes on the measured inputs"""
    for n in ONE_SIZES:
        assert eng.basepoint_tables_mul(handles[1], x.ss[:32 * n], None, n) == eng.mul_batch(x.ss[:32 * n], n, x.pts[:32], 1, n)[1]
    for k in MANY_KS:
        want = eng.mul_batch(x.ss, N_BIG, x.per_item[k], N_BIG, N_BIG)[1]
        for v in (1, 0):
            eng.set_option("bpt_group", v)
            assert eng.basepoint_tables_mul(handles[k], x.ss, x.idx_b[k], N_BIG) == want
    eng.set_option("bpt_group", 1)


def profile_kernels(out_path, calls):
    """kernel name -> device ms per call of each configuration, with torch.profiler (run in a process of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import curve25519_dalek_b200 as pkg
    eng = pkg.Engine(0)
    x = Inputs(eng)
    handles = {k: eng.basepoint_tables_new(x.pts[:32 * k], k)[1] for k in set(MANY_KS) | {1}}
    res = {}
    for name, fn in configs(eng, x, handles).items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
        ker = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0 and not e.key.startswith("Memcpy") and not e.key.startswith("Memset"):
                ker[e.key[:80]] = round(t / 1e3 / calls, 4)
        res[name] = ker
    for h in handles.values():
        eng.basepoint_tables_destroy(h)
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
    x = Inputs(eng)
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "calls": a.calls, "warmup": a.warmup}

    def new_call(k):
        _, h, _ = eng.basepoint_tables_new(x.pts[:32 * k], k)
        ms = eng.last_call_ms()
        eng.basepoint_tables_destroy(h)
        return ms
    for k in NEW_KS:
        for _ in range(a.warmup):
            new_call(k)
        res["new_k%d_ms" % k] = statistics.median(new_call(k) for _ in range(a.calls))
    handles = {k: eng.basepoint_tables_new(x.pts[:32 * k], k)[1] for k in set(MANY_KS) | {1}}
    check_outputs(eng, x, handles)
    cfg = configs(eng, x, handles)
    names = list(cfg)
    for pair in groups(names):                             # each group alternated call by call
        times = {p: [] for p in pair}
        for _ in range(a.warmup):
            for p in pair:
                cfg[p]()
        for _ in range(a.calls):
            for p in pair:
                cfg[p]()
                times[p].append(eng.last_call_ms())
        for p in pair:
            ms = statistics.median(times[p])
            n = int(p.rsplit("_", 1)[1]) if not p.split("_")[-1].startswith("k") else N_BIG
            res[p + "_ms"] = round(ms, 4)
            res[p + "_per_s"] = round(n / ms * 1e3)
    for h in handles.values():
        eng.basepoint_tables_destroy(h)
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
