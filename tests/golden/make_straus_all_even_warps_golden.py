"""Writes tests/golden/straus_all_even_warps.json: the two MSMs on which tools/bench_msm_batch.py once found the single
vartime call disagreeing with the oracle (16384x64 sample 24 and ragged_8192 sample 41).  Both run on the vartime Straus
path (fewer than 190 terms) and both hold a warp of at least five terms whose scalars are all even -- the case where the
warp's last doubling skipped T and the warp sum then read a stale T.

The inputs are regenerated in the benchmark's order, on the CPU:
  * random.Random(1) draws 4096 pool scalars; pool point i = pool_scalar_i * B;
  * the same generator then draws 4096 scalars per (shape, format) in the benchmark's shapes() order:
    262144x4, 65536x16, 16384x64, 4096x256 (compressed, extended, ristretto), 1024x1024, ragged_8192;
  * term i of MSM j takes the scalar and the pool point at index (offs[j] + i) mod 4096;
  * the 64 sampled MSMs of a shape are random.Random(9).sample(range(m), 64).
Each record holds the scalars, the compressed points and the oracle's result.  Run from the repository root:
python tests/golden/make_straus_all_even_warps_golden.py"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))

POOL = 4096
RECORDED = (("16384x64", 24, 3), ("ragged_8192", 41, 13))     # shape, sample index, the all-even warp


def shapes():
    rnd = random.Random(5)
    return {"262144x4": [4] * (1 << 18), "65536x16": [16] * (1 << 16), "16384x64": [64] * (1 << 14), "4096x256": [256] * 4096,
            "1024x1024": [1024] * 1024, "ragged_8192": [rnd.randrange(1, 513) for _ in range(8192)]}


def all_even_warps(scalars):
    """warps (8 terms each) with at least five terms, all of them even"""
    return [w for w in range((len(scalars) + 7) // 8)
            if len(scalars[8 * w:8 * w + 8]) >= 5 and all(v % 2 == 0 for v in scalars[8 * w:8 * w + 8])]


def main():
    import oracle_lib
    import pyref
    orc = oracle_lib.load()
    rnd = random.Random(1)
    pool_scalars = [rnd.randrange(pyref.L) for _ in range(POOL)]
    draws = {}
    for key, sizes in shapes().items():
        for fmt in (("compressed", "extended", "ristretto") if key == "4096x256" else ("compressed",)):
            draws[(key, fmt)] = [rnd.randrange(pyref.L) for _ in range(POOL)]
    B = orc.basepoint()
    pool_points = {}

    def point(i):
        if i not in pool_points:
            pool_points[i] = orc.scalarmul(pool_scalars[i].to_bytes(32, "little"), B)
        return pool_points[i]

    cases = []
    for key, sample, warp in RECORDED:
        sizes = shapes()[key]
        j = random.Random(9).sample(range(len(sizes)), 64)[sample]
        off = sum(sizes[:j])
        idx = [(off + i) % POOL for i in range(sizes[j])]
        scalars = [draws[(key, "compressed")][k] for k in idx]
        assert len(scalars) < 190                                  # the Straus path
        assert all_even_warps(scalars) == [warp], (key, all_even_warps(scalars))
        points = [point(k) for k in idx]
        sb = [v.to_bytes(32, "little") for v in scalars]
        want = orc.msm("optional", sb, points)
        assert orc.compress(want) == orc.compress(orc.msm("straus_vartime", sb, points))
        cases.append({"shape": key, "sample_index": sample, "msm_index": j, "terms": len(scalars), "all_even_warp": warp,
                      "scalars": [s.hex() for s in sb], "points": [orc.compress(P).hex() for P in points],
                      "expected": orc.compress(want).hex()})
    with open(os.path.join(ROOT, "tests", "golden", "straus_all_even_warps.json"), "w") as f:
        json.dump({"source": "tests/golden/make_straus_all_even_warps_golden.py", "cases": cases}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
