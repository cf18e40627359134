"""Call time of dalek_b200_ristretto_vartime_msm from pinned host buffers, per size: below 190 pairs the call runs vartime
Straus, from 2^18 pairs the inputs are streamed in chunks, in between it is the bucket pipeline in one piece.  The points
are a_i G + b_i H of the engine's own double-base batch (G the Ristretto basepoint), the scalars uniform below 2^252.

Every build named with --lib NAME=PATH runs in a process of its own (DALEK_B200_LIB), the builds alternated, --rounds
times.  Per size and build: the median of --calls calls after --warmup calls in each round, then the median, minimum and
maximum of the round medians.  The results of all builds must be byte-equal.  Prints one JSON document and writes it to
--out if given.

usage: python tools/bench_ristretto_msm.py [--lib NAME=PATH ...] [--rounds 3] [--calls 21] [--warmup 3] [--sizes N ...]
                                           [--set OPTION=VALUE ...] [--out FILE]"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIZES = [1, 17, 189, 190, 1000, 1 << 16, 1 << 18, 1 << 20]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, sm, sm_max = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def child(a):
    """one build: {n: {ms, launches, result}} on stdout"""
    import numpy as np
    import torch
    import bench
    import curve25519_dalek_b200 as pkg
    eng = pkg.Engine(0)
    for s in a.set:
        name, value = s.split("=", 1)
        eng.set_option(name, int(value))
    nmax = max(a.sizes)
    G = bytes.fromhex("e2f2ae0a6abc4e71a884a961c500515f58e30b6aa582dd8db6a65945e08d2d76")   # constants.rs:57-60
    h = np.frombuffer(hashlib.sha512(b"dalek-b200/H").digest()[:32], dtype=np.uint8).copy(); h[31] &= 0x0F
    rc, H = eng.ristretto_double_base_batch(np.zeros(32, dtype=np.uint8), h, G, G, 1)
    assert rc == 0
    pts = torch.empty(32 * nmax, dtype=torch.uint8).pin_memory()
    rc, _ = eng.ristretto_double_base_batch(bench.fast_scalars(nmax, seed=41), bench.fast_scalars(nmax, seed=42), G, H, nmax, out=pts)
    assert rc == 0
    scalars = torch.from_numpy(bench.fast_scalars(nmax, seed=43).reshape(-1)).pin_memory()
    out = np.zeros(32, dtype=np.uint8)
    res = {}
    for n in a.sizes:
        def call():
            rc = eng.lib.dalek_b200_ristretto_vartime_msm(eng.h, scalars.data_ptr(), pts.data_ptr(), n, out.ctypes.data)
            if rc != 0:
                raise SystemExit("ristretto_vartime_msm failed on valid points (rc=%d)" % rc)
        for _ in range(a.warmup):
            call()
        l0 = eng.launch_count()
        call()
        launches = eng.launch_count() - l0
        ms = []
        for _ in range(a.calls):
            t = time.perf_counter()
            call()
            ms.append((time.perf_counter() - t) * 1e3)
        res[n] = {"ms": statistics.median(ms), "launches": launches, "result": out.tobytes().hex()}
    eng.close()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build to time (default: this tree's build)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=SIZES)
    ap.add_argument("--set", action="append", default=[], metavar="OPTION=VALUE", help="an engine option for every build")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)
    libs = [s.split("=", 1) for s in a.lib] or [["this", os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")]]
    rounds = {name: [] for name, _ in libs}
    for _ in range(a.rounds):
        for name, path in libs:
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--calls", str(a.calls), "--warmup", str(a.warmup),
                   "--sizes"] + [str(n) for n in a.sizes] + ["--set=" + s for s in a.set]
            r = subprocess.run(cmd, env=dict(os.environ, DALEK_B200_LIB=os.path.abspath(path)), capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit("%s failed:\n%s" % (name, r.stderr))
            rounds[name].append({int(k): v for k, v in json.loads(r.stdout.splitlines()[-1]).items()})
    doc = dict(gpu_info(), path="pinned host buffers, blocking call", options=a.set, calls=a.calls, warmup=a.warmup,
               rounds=a.rounds, results={})
    for n in a.sizes:
        results = {rs[n]["result"] for name in rounds for rs in rounds[name]}
        if len(results) != 1:
            raise SystemExit("results differ at n = %d: %s" % (n, sorted(results)))
        row = {}
        for name in rounds:
            med = [rs[n]["ms"] for rs in rounds[name]]
            row[name] = {"ms_median": statistics.median(med), "ms_min": min(med), "ms_max": max(med),
                         "launches": rounds[name][-1][n]["launches"]}
        doc["results"][str(n)] = row
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
