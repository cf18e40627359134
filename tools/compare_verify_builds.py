"""Call every Ed25519 verify entry point of two builds of libdalek_b200.so on the same seeded inputs and check that they
agree: return codes, per-batch verdicts, per-signature results, last_zs and the number of kernel launches of each call.

    python tools/compare_verify_builds.py --base OTHER/libdalek_b200.so [--out DIR]

compares the in-tree build with OTHER.  The engine loads one library per process (DALEK_B200_LIB), so each build runs
in a process of its own (`--run FILE` writes one build's records).  Sizes 0, 1, 300 and 2^18 + 5 (host buffers of
2^18 or more signatures are streamed in pieces), the options dedupe_keys in {0, 1} and verify_chunk in {0, 64}, valid
signatures and the same with a non-canonical s, an undecodable R and an undecodable key planted.  Needs an H100."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [0, 1, 300, (1 << 18) + 5]
NKEYS = 61
CONTEXT = b"compare"


def make_inputs(eng, n, bad):
    seeds_k = np.frombuffer(b"".join(hashlib.sha512(b"cmp%d" % k).digest()[:32] for k in range(NKEYS)), dtype=np.uint8)
    seeds = np.ascontiguousarray(seeds_k.reshape(NKEYS, 32)[np.arange(n) % NKEYS])
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum((np.arange(n) % 7) * 11)
    rng = np.random.Generator(np.random.PCG64(n))
    fl = rng.integers(0, 256, size=int(offs[-1]) + 1, dtype=np.uint8)
    phs = rng.integers(0, 256, size=64 * n + 1, dtype=np.uint8)
    if n:
        pks, sigs = eng.sign_batch_flat(seeds, fl, offs, n)
        rc, ph_sigs = eng.sign_prehashed(seeds, n, phs, n, context=CONTEXT)
        assert rc == 0
    else:
        pks, sigs, ph_sigs = b"", b"", b""
    sg = np.frombuffer(sigs + b"\0", dtype=np.uint8).copy()
    ph_sg = np.frombuffer(ph_sigs + b"\0", dtype=np.uint8).copy()
    pk = np.frombuffer(pks + b"\0", dtype=np.uint8).copy()
    if bad and n:
        i_s, i_r, i_k = n // 3, (2 * n) // 3, n - 1
        for s in (sg, ph_sg):
            s[64 * i_s + 63] |= 0xf0                                                    # s >= l
            s[64 * i_r:64 * i_r + 32] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)   # undecodable R
        pk[32 * i_k:32 * i_k + 32] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)       # undecodable key
    kp = np.zeros(20, dtype=np.uint64)
    if n:                                                   # the planted key decodes to nothing: its limbs are what the codec left
        _, limbs, _ = eng.decompress_batch(pk.tobytes(), n)
        kp = np.frombuffer(limbs, dtype=np.uint64).copy()
    return {"msgs": fl, "offs": offs, "sigs": sg, "keys": pk, "kp": kp, "ph": phs, "ph_sigs": ph_sg}


def entry_points(eng, inp, dev, n):
    """name -> call() returning (rc, verdicts or results or None, is a verify_batch[es] call)"""
    L, h = eng.lib, eng.h
    hp = {k: v.ctypes.data for k, v in inp.items()}
    dp = {k: v.data_ptr() for k, v in dev.items()}
    bs = 16 if n < 4096 else 256
    nb = (n + bs - 1) // bs
    verdicts = (C.c_int32 * max(nb, 1))()
    results = (C.c_uint8 * max(n, 1))()
    ptrs = np.ascontiguousarray(inp["msgs"].ctypes.data + inp["offs"][:n]).astype(np.uint64)
    lens = np.diff(inp["offs"]).astype(np.uint64)
    keep = (ptrs, lens)
    V = lambda: list(verdicts)[:nb]
    R = lambda: bytes(results)[:n]

    def batch(fn, *a):
        return lambda: (fn(h, *a), None, True)

    def batches(fn, *a):
        return lambda: (fn(h, *a, bs, C.addressof(verdicts)), V(), True)

    def each(fn, *a):
        return lambda: (fn(h, *a, C.addressof(results)), R(), False)

    return keep, {
        "verify_batch": batch(L.ed25519_b200_verify_batch, ptrs.ctypes.data, lens.ctypes.data, hp["sigs"], hp["keys"], n),
        "verify_batch_flat": batch(L.ed25519_b200_verify_batch_flat, hp["msgs"], hp["offs"], hp["sigs"], hp["keys"], n),
        "verify_batch_flat_dev": batch(L.ed25519_b200_verify_batch_flat_dev, dp["msgs"], dp["offs"], dp["sigs"], dp["keys"], n, 0),
        "verify_batch_flat_points": batch(L.ed25519_b200_verify_batch_flat_points, hp["msgs"], hp["offs"], hp["sigs"], hp["keys"], hp["kp"], n),
        "verify_batch_flat_points_dev": batch(L.ed25519_b200_verify_batch_flat_points_dev, dp["msgs"], dp["offs"], dp["sigs"], dp["keys"],
                                              dp["kp"], n),
        "verify_batches_flat": batches(L.ed25519_b200_verify_batches_flat, hp["msgs"], hp["offs"], hp["sigs"], hp["keys"], n),
        "verify_batches_flat_dev": batches(L.ed25519_b200_verify_batches_flat_dev, dp["msgs"], dp["offs"], dp["sigs"], dp["keys"], n),
        "verify_batches_flat_points": batches(L.ed25519_b200_verify_batches_flat_points, hp["msgs"], hp["offs"], hp["sigs"], hp["keys"],
                                              hp["kp"], n),
        "verify_batches_flat_points_dev": batches(L.ed25519_b200_verify_batches_flat_points_dev, dp["msgs"], dp["offs"], dp["sigs"],
                                                  dp["keys"], dp["kp"], n),
        "verify_each_flat": each(L.ed25519_b200_verify_each_flat, hp["msgs"], hp["offs"], hp["sigs"], hp["keys"], n, 0),
        "verify_each_flat_dev": each(L.ed25519_b200_verify_each_flat_dev, dp["msgs"], dp["offs"], dp["sigs"], dp["keys"], n, 1),
        "verify_prehashed_each": each(L.ed25519_b200_verify_prehashed_each, hp["ph"], CONTEXT, len(CONTEXT), hp["ph_sigs"], hp["keys"], n, 0),
    }


def run(out_path):
    import torch
    sys.path.insert(0, ROOT)
    import curve25519_dalek_b200 as pkg
    eng = pkg.Engine(0)
    records = {}
    for n in SIZES:
        for bad in (False, True):
            inp = make_inputs(eng, n, bad)
            dev = {k: torch.from_numpy(v if v.dtype == np.uint8 else v.view(np.int64)).cuda() for k, v in inp.items()}
            torch.cuda.synchronize()
            keep, calls = entry_points(eng, inp, dev, n)
            for dedupe in (0, 1):
                for chunk in (0, 64):
                    eng.set_option("dedupe_keys", dedupe)
                    eng.set_option("verify_chunk", chunk)
                    for name, call in calls.items():
                        l0 = eng.launch_count()
                        rc, out, is_batch = call()
                        rec = {"rc": rc, "launches": eng.launch_count() - l0}
                        if isinstance(out, bytes):
                            rec["results_sha256"] = hashlib.sha256(out).hexdigest()
                            rec["failed"] = int(sum(1 for r in out if r))
                        elif out is not None:
                            rec["verdicts"] = out
                        if is_batch and rc >= 0:
                            rec["zs_sha256"] = hashlib.sha256(eng.last_zs(n)).hexdigest()
                        records["%s|n=%d|%s|dedupe=%d|chunk=%d" % (name, n, "planted" if bad else "valid", dedupe, chunk)] = rec
            del keep
    eng.set_option("dedupe_keys", 1)
    eng.set_option("verify_chunk", 0)
    with open(out_path, "w") as f:
        json.dump(records, f, indent=1, sort_keys=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--base", help="the other build's libdalek_b200.so")
    ap.add_argument("--out", default="compare_verify_out", help="directory for the two builds' records")
    ap.add_argument("--run", metavar="FILE", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        return run(args.run)
    if not args.base:
        ap.error("--base is required")
    os.makedirs(args.out, exist_ok=True)
    got = {}
    for tag, lib in (("base", os.path.abspath(args.base)), ("tree", None)):
        env = dict(os.environ)
        env.pop("DALEK_B200_LIB", None)
        if lib:
            env["DALEK_B200_LIB"] = lib
        path = os.path.join(args.out, "verify_records_%s.json" % tag)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--run", path], env=env, check=True)
        with open(path) as f:
            got[tag] = json.load(f)
    base, tree = got["base"], got["tree"]
    diff = sorted(k for k in set(base) | set(tree) if base.get(k) != tree.get(k))
    for k in diff[:20]:
        print("MISMATCH %s\n  base %s\n  tree %s" % (k, base.get(k), tree.get(k)))
    print(json.dumps({"calls": len(tree), "mismatches": len(diff),
                      "return_codes": sorted({r["rc"] for r in tree.values()})}))
    return 1 if diff else 0


if __name__ == "__main__":
    sys.exit(main() or 0)
