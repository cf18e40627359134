"""Device memory footprint of one engine context after a fixed sequence of 2^20-item calls across the entry-point
families: the drop in free device memory (torch.cuda.mem_get_info, i.e. cudaMemGetInfo) from before dalek_b200_init to
after the last call, and from there to after dalek_b200_destroy.  The context's workspaces grow on demand and are kept
until the context is destroyed, so the first figure is what the sequence leaves allocated.  Every input is made on the
GPU by the engine itself (basepoint multiples, signatures), so the calls run their full paths.  Prints one JSON object.

usage: python tools/ws_footprint.py [--n 1048576] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import curve25519_dalek_b200 as pkg
    n = a.n
    gen = np.random.Generator(np.random.PCG64(7))
    scalars = gen.integers(0, 256, size=(n, 32), dtype=np.uint8)
    scalars[:, 31] &= 0x7f                                     # bit 255 clear (Scalar invariant #1)
    seeds = gen.integers(0, 256, size=(n, 32), dtype=np.uint8).tobytes()
    msgs = gen.integers(0, 256, size=(n, 32), dtype=np.uint8).tobytes()
    offsets = (np.arange(n + 1, dtype=np.uint64) * 32).tobytes()
    wide = gen.integers(0, 256, size=(n, 64), dtype=np.uint8).tobytes()
    lizard = gen.integers(0, 256, size=(n, 16), dtype=np.uint8).tobytes()
    ab = np.concatenate([scalars, scalars[::-1]], axis=1).tobytes()
    sc = scalars.tobytes()
    torch.cuda.init()
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    eng = pkg.Engine(0)
    _, points = eng.mul_base_batch(sc, n)                      # valid compressed points
    steps = []

    def run(name, fn):
        try:
            fn()
            steps.append(name)
        except pkg.EngineError as e:                            # a rejected input still counts as a step taken
            steps.append("%s (%s)" % (name, e))

    run("edwards_vartime_msm", lambda: eng.edwards_vartime_msm(sc, points, n))
    run("edwards_ct_msm", lambda: eng.edwards_ct_msm(sc, points, n))
    run("partial+combine", lambda: eng.edwards_msm_combine(eng.edwards_msm_partial(sc, points, n, n)[1], 1, n))
    m = n // 64
    run("msm_batch", lambda: eng.msm_batch(sc, points, (np.arange(m + 1, dtype=np.uint64) * 64).tobytes(), m))
    pks = eng.verifying_keys(seeds, n)
    sigs = eng.sign_flat(seeds, n, msgs, offsets, n)
    steps += ["verifying_keys", "sign_flat"]
    run("verify_batch_flat", lambda: eng.verify_batch_flat(msgs, offsets, sigs, pks, n))
    run("verify_batches_flat", lambda: eng.verify_batches_flat(msgs, offsets, sigs, pks, n, 64))
    run("verify_each_flat", lambda: eng.verify_each_flat(msgs, offsets, sigs, pks, n))
    run("x25519_batch", lambda: eng.x25519_batch(sc, points, n))
    run("montgomery_mul_batch", lambda: eng.montgomery_mul_batch(sc, n, points, n, n))
    run("mul_batch", lambda: eng.mul_batch(sc, n, points, n, n))
    run("vartime_double_base_batch", lambda: eng.vartime_double_base_batch(ab, points, n))
    run("decompress_batch", lambda: eng.decompress_batch(points, n))
    run("scalar_from_wide_batch", lambda: eng.scalar_from_wide_batch(wide, n))
    run("scalar_invert_batch", lambda: eng.scalar_invert_batch(sc, n))
    run("ristretto_hash_from_bytes_batch", lambda: eng.ristretto_hash_from_bytes_batch(msgs, offsets, n))
    run("ristretto_lizard_encode_batch", lambda: eng.ristretto_lizard_encode_batch(lizard, n))
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    eng.close()
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info()
    res = dict(gpu_info(), n=n, total_bytes=total, footprint_bytes=free0 - free1, footprint_mib=round((free0 - free1) / 2**20, 1),
               left_after_destroy_bytes=free0 - free2, steps=steps)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
