"""Throughput of batched independent MSMs (dalek_b200_msm_batch) on the GPU, with the comparisons measured in the same
run; prints one JSON line.

  shapes        m x n: 2^18 x 4, 2^16 x 16, 2^14 x 64, 4096 x 256, 1024 x 1024 and a ragged mix (sizes 1..512 from a seed),
                variable time and constant time, host buffers (copies included) and device buffers, CompressedEdwardsY;
                4096 x 256 also from extended limbs and CompressedRistretto
  *_call_ms     median device span of the call (CUDA events, dalek_b200_last_call_ms); *_host_ms the median host clock
                around the blocking call
  single_loop   the same MSMs as a loop of single calls on a 64-MSM SAMPLE of the shape (host clock), alternating with
                the batched call on the same sample
  cpu_oracle    the C oracle on the same sample, one core and one thread per core
Outputs of the batched call, the single calls and the oracle are compared on the sample before anything is timed; a
single call that disagrees with the batched call is checked against the oracle and listed in the result.

--ab NAME=LIB[,NAME=LIB...] instead times 4096 x 256 and 2^18 x 4 from device buffers with each alternative build of the
library (one engine each, calls alternating), for the chunk-length A/B.

usage: python tools/bench_msm_batch.py [--calls 21] [--warmup 2] [--out FILE] [--ab 8=build/libmb8.so,...]"""
import argparse
import array
import concurrent.futures
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
POOL = 4096


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def shapes():
    rnd = random.Random(5)
    return {"262144x4": [4] * (1 << 18), "65536x16": [16] * (1 << 16), "16384x64": [64] * (1 << 14), "4096x256": [256] * 4096,
            "1024x1024": [1024] * 1024, "ragged_8192": [rnd.randrange(1, 513) for _ in range(8192)]}


def offsets_of(sizes):
    offs = array.array("Q", [0])
    for n in sizes:
        offs.append(offs[-1] + n)
    return offs


def timed(fn, eng, calls, warmup):
    for _ in range(warmup):
        fn()
    dev, host = [], []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        host.append((time.perf_counter() - t) * 1e3)
        dev.append(eng.last_call_ms())
    return statistics.median(dev), statistics.median(host)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--ab", default=None)
    a = ap.parse_args()
    import torch
    import curve25519_dalek_b200 as pkg
    import oracle_lib
    import pyref
    if not torch.cuda.is_available():
        raise SystemExit("bench_msm_batch needs a GPU")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "calls": a.calls, "warmup": a.warmup}
    eng = pkg.Engine(0)
    orc = oracle_lib.load()
    rnd = random.Random(1)
    limbs, comp = eng.mul_base_batch(b"".join(rnd.randrange(pyref.L).to_bytes(32, "little") for _ in range(POOL)), POOL)
    limbs = bytes(limbs)
    rist = b"".join(orc.ristretto_compress(orc.decompress(comp[32 * i:32 * i + 32])) for i in range(POOL))
    points = {COMPRESSED: (comp, 32), EXTENDED: (limbs, 160), RISTRETTO: (rist, 32)}

    def inputs(sizes, fmt=COMPRESSED):
        total = sum(sizes)
        s = b"".join(rnd.randrange(pyref.L).to_bytes(32, "little") for _ in range(POOL)) * (total // POOL + 1)
        p, w = points[fmt]
        return s[:32 * total], (p * (total // POOL + 1))[:w * total], offsets_of(sizes)

    def dev(b):
        return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()

    if a.ab:
        engines = {"tree": eng}
        for item in a.ab.split(","):
            k, path = item.split("=")
            os.environ["DALEK_B200_LIB"] = os.path.join(ROOT, path)
            pkg.engine._lib = None
            engines[k] = pkg.Engine(0)
        res["ab"] = {}
        for key in ("4096x256", "262144x4"):
            sizes = shapes()[key]
            s, p, offs = inputs(sizes)
            d = (dev(s), dev(p), dev(offs.tobytes()))
            for ct in (False, True):
                outs, times = {}, {k: [] for k in engines}
                for k, e in engines.items():
                    outs[k] = e.msm_batch(*d, len(sizes), constant_time=ct, device_ptrs=True)[:3]
                assert all(o == outs["tree"] for o in outs.values())
                for _ in range(a.calls):
                    for k, e in engines.items():
                        e.msm_batch(*d, len(sizes), constant_time=ct, device_ptrs=True)
                        times[k].append(e.last_call_ms())
                res["ab"]["%s_%s" % (key, "ct" if ct else "vt")] = {k: statistics.median(v) for k, v in times.items()}
    else:
        cores = os.cpu_count() or 1
        res["cpu_cores"] = cores
        for key, sizes in shapes().items():
            m, total = len(sizes), sum(sizes)
            fmts = (COMPRESSED, EXTENDED, RISTRETTO) if key == "4096x256" else (COMPRESSED,)
            for fmt in fmts:
                s, p, offs = inputs(sizes, fmt)
                d = (dev(s), dev(p), dev(offs.tobytes()))
                w = points[fmt][1]
                for ct in (False, True):
                    tag = "%s_%s_%s" % (key, ("compressed", "extended", "ristretto")[fmt], "ct" if ct else "vt")
                    rc, out, ok, _ = eng.msm_batch(s, p, offs.tobytes(), m, fmt, constant_time=ct)
                    assert rc == 0 and eng.msm_batch(*d, m, fmt, constant_time=ct, device_ptrs=True)[:3] == (rc, out, ok)
                    # the 64-MSM sample: batched call, loop of single calls and the oracle give the same bytes
                    pick = random.Random(9).sample(range(m), 64)
                    seg = [(s[32 * offs[j]:32 * offs[j + 1]], p[w * offs[j]:w * offs[j + 1]], offs[j + 1] - offs[j]) for j in pick]
                    ss, sp = b"".join(x[0] for x in seg), b"".join(x[1] for x in seg)
                    so = offsets_of([x[2] for x in seg]).tobytes()

                    def single(x):
                        if fmt == RISTRETTO:
                            return eng.ristretto_vartime_msm(x[0], x[1], x[2])[1]
                        return (eng.edwards_ct_msm if ct else eng.edwards_vartime_msm)(x[0], x[1], x[2], point_fmt=fmt)[1]
                    have_single = not (ct and fmt == RISTRETTO)
                    sample_out = eng.msm_batch(ss, sp, so, 64, fmt, constant_time=ct)[1]
                    assert sample_out == b"".join(out[32 * j:32 * j + 32] for j in pick)
                    if have_single:
                        singles = [single(x) for x in seg]
                        diff = [(k, seg[k][2]) for k in range(64) if singles[k] != sample_out[32 * k:32 * k + 32]]
                        for k, n in diff:          # the oracle decides; a disagreeing single call is recorded, not timed around
                            x = seg[k]
                            pts_k = [orc.decompress(x[1][32 * i:32 * i + 32]) for i in range(n)]
                            scal_k = [x[0][32 * i:32 * i + 32] for i in range(n)]
                            want = orc.compress(orc.msm_ct(scal_k, pts_k) if ct else orc.msm("optional", scal_k, pts_k))
                            assert want == sample_out[32 * k:32 * k + 32], (tag, k)
                            res.setdefault("single_call_disagrees_with_oracle", []).append({"shape": tag, "sample_index": k, "terms": n})
                    dms, hms = timed(lambda: eng.msm_batch(*d, m, fmt, constant_time=ct, device_ptrs=True), eng, a.calls, a.warmup)
                    res[tag + "_dev"] = {"call_ms": dms, "host_ms": hms, "msms_per_s": m / dms * 1e3, "terms_per_s": total / dms * 1e3}
                    dms, hms = timed(lambda: eng.msm_batch(s, p, offs.tobytes(), m, fmt, constant_time=ct), eng, a.calls, a.warmup)
                    res[tag + "_host"] = {"call_ms": dms, "host_ms": hms, "msms_per_s": m / hms * 1e3, "terms_per_s": total / hms * 1e3}
                    if fmt != COMPRESSED:
                        continue
                    # sample: batched call against the loop of single calls, alternating; then the oracle
                    tb, tl = [], []
                    for _ in range(5):
                        t = time.perf_counter(); eng.msm_batch(ss, sp, so, 64, fmt, constant_time=ct); tb.append(time.perf_counter() - t)
                        t = time.perf_counter(); [single(x) for x in seg]; tl.append(time.perf_counter() - t)
                    res[tag + "_sample64"] = {"batched_ms": statistics.median(tb) * 1e3, "single_loop_ms": statistics.median(tl) * 1e3,
                                              "single_loop_whole_shape_ms_extrapolated": statistics.median(tl) * 1e3 * m / 64}
                    pts = [[orc.decompress(x[1][32 * i:32 * i + 32]) for i in range(x[2])] for x in seg]
                    scal = [[x[0][32 * i:32 * i + 32] for i in range(x[2])] for x in seg]

                    def cpu(j):
                        r = orc.msm_ct(scal[j], pts[j]) if ct else orc.msm("optional", scal[j], pts[j])
                        return orc.compress(r)
                    t = time.perf_counter(); got = [cpu(j) for j in range(64)]; one = time.perf_counter() - t
                    assert b"".join(got) == sample_out
                    with concurrent.futures.ThreadPoolExecutor(cores) as ex:
                        t = time.perf_counter(); list(ex.map(cpu, range(64))); pool = time.perf_counter() - t
                    res[tag + "_cpu_oracle_sample64"] = {"one_core_msms_per_s": 64 / one, "all_cores_msms_per_s": 64 / pool}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
