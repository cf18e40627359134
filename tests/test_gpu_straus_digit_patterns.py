"""The vartime Straus path of the engine (csrc/straus_vt.cu, every vartime MSM below 190 terms) at scalar patterns that
are uniform across a warp (tests/straus_patterns.py): all-even warps, shared trailing zero digits, warps with no
doubling, all-zero warps, even scalars with bit 255 set, small-order points in an all-even warp.  Each call --
edwards_vartime_msm from host and device buffers, compressed and extended (Z != 1) points, and ristretto_vartime_msm --
is compared with the oracle on the Straus path and on the bucket path (option small_straus = 0).  Then the two recorded
benchmark inputs whole, and a few thousand MSMs with mostly-even scalars, single calls against one msm_batch call."""
import array
import json
import os
import random

import pytest

import point_checks
import pyref
import straus_patterns as sp

pytestmark = pytest.mark.gpu

COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
NS = (5, 8, 9, 13, 16, 64, 150, 181, 189)
PATTERNS = ("even",) + tuple("pow2_%d" % k for k in sp.K_TRAILING) + ("even_bit255", "ones", "small_odd", "zero", "small_order")


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def pool(oracle):
    """189 random points: oracle points, compressed, extended limbs with Z != 1, Ristretto encodings."""
    rnd = random.Random(77)
    pts = sp.random_points(oracle, rnd, 189)
    ext = []
    for P in pts:
        q = oracle.sub(oracle.add(oracle.double(P), P), oracle.double(P))
        ext.append(b"".join(int(v).to_bytes(8, "little") for v in oracle.p3_limbs(q)))
    return {"pts": pts, "comp": [oracle.compress(P) for P in pts], "ext": ext,
            "rist": [oracle.ristretto_compress(P) for P in pts], "small": sp.small_order_points(oracle)}


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf) or bytearray(8), dtype=torch.uint8).cuda()


def placements(nw):
    """which warps follow the pattern: first, last, middle, every"""
    return {"first": [0], "last": [nw - 1], "middle": [nw // 2], "every": list(range(nw))}


def make_case(oracle, pool, n, pattern, where, rnd):
    """scalars (ints) and points of one call: the placed warps follow `pattern`, the others hold random scalars.
    `small_order` is an all-even warp whose points include the identity and small-order points; `zero` keeps at least
    one live warp around the zero warp(s)."""
    nw = (n + 7) // 8
    warps = placements(nw)[where]
    pat = {"small_order": "even"}.get(pattern, pattern)
    scalars = []
    for w in range(nw):
        cnt = min(8, n - 8 * w)
        scalars += sp.pattern_scalars(pat, rnd, cnt) if w in warps else [rnd.randrange(pyref.L) for _ in range(cnt)]
    idx = list(range(n))
    rnd.shuffle(idx)
    pts = [pool["pts"][i] for i in idx]
    small = set()
    if pattern == "small_order":
        for w in warps:
            for g, P in enumerate(pool["small"]):
                if 8 * w + 2 * g < n:
                    pts[8 * w + 2 * g] = P
                    small.add(8 * w + 2 * g)
    if pattern == "zero" and where == "every":
        scalars[-1] = rnd.randrange(pyref.L)                        # one live term
    return scalars, pts, idx, small


def run_all_forms(eng, oracle, pool, scalars, pts, idx, small, what):
    n = len(scalars)
    want_pt = sp.msm_exact(oracle, scalars, pts)
    want = oracle.compress(want_pt)
    sb = b"".join(v.to_bytes(32, "little") for v in scalars)
    comp = b"".join(oracle.compress(P) for P in pts)
    ext = b"".join(pool["ext"][i] if j not in small else
                   b"".join(int(v).to_bytes(8, "little") for v in oracle.p3_limbs(pts[j]))
                   for j, i in enumerate(idx))
    rist = None if small else b"".join(pool["rist"][i] for i in idx)
    for straus in (1, 0):
        eng.set_option("small_straus", straus)
        try:
            l0 = eng.launch_count()
            rc, got, limbs = eng.edwards_vartime_msm(sb, comp, n, point_fmt=COMPRESSED, want_limbs=True)
            launches = eng.launch_count() - l0
            assert rc == 0 and got == want, (what, straus, "compressed")
            assert (launches <= 5) == bool(straus), (what, launches)
            point_checks.check_limbs(limbs, want, what=(what, straus))
            rc, got, _ = eng.edwards_vartime_msm(sb, ext, n, point_fmt=EXTENDED)
            assert rc == 0 and got == want, (what, straus, "extended")
            for fmt, buf in ((COMPRESSED, comp), (EXTENDED, ext)):
                rc, got, limbs = eng.edwards_vartime_msm(dev(sb), dev(buf), n, point_fmt=fmt, device_ptrs=True, want_limbs=True)
                assert rc == 0 and got == want, (what, straus, "dev", fmt)
                point_checks.check_limbs(limbs, want, what=(what, straus, "dev", fmt))
            if rist is not None:
                rc, got = eng.ristretto_vartime_msm(sb, rist, n)
                assert rc == 0 and got == oracle.ristretto_compress(want_pt), (what, straus, "ristretto")
        finally:
            eng.set_option("small_straus", 1)


@pytest.mark.parametrize("n", NS)
def test_warp_uniform_patterns(eng, oracle, pool, n):
    """Every pattern of straus_patterns.py in the first, last, middle and every warp, at n = 5 .. 189."""
    rnd = random.Random(1000 + n)
    nw = (n + 7) // 8
    for pattern in PATTERNS:
        for where in placements(nw):
            if pattern == "zero" and nw == 1:
                continue
            scalars, pts, idx, small = make_case(oracle, pool, n, pattern, where, rnd)
            run_all_forms(eng, oracle, pool, scalars, pts, idx, small, (n, pattern, where))


def golden_cases():
    with open(os.path.join(os.path.dirname(__file__), "golden", "straus_all_even_warps.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["shape"])
def test_recorded_benchmark_inputs(eng, oracle, case):
    """The two MSMs (64 and 181 terms) on which the single vartime call once disagreed with the oracle: each holds a
    warp whose scalars are all even.  Single calls in every point format, host and device, and msm_batch."""
    n = case["terms"]
    sb = b"".join(bytes.fromhex(x) for x in case["scalars"])
    comp = b"".join(bytes.fromhex(x) for x in case["points"])
    want = bytes.fromhex(case["expected"])
    pts = [oracle.decompress(bytes.fromhex(x)) for x in case["points"]]
    assert oracle.compress(oracle.msm("straus_vartime", [bytes.fromhex(x) for x in case["scalars"]], pts)) == want
    ext = b"".join(b"".join(int(v).to_bytes(8, "little") for v in oracle.p3_limbs(oracle.sub(oracle.add(oracle.double(P), P), oracle.double(P))))
                   for P in pts)                                   # (2P + P) - 2P: the same point, Z != 1
    rist = b"".join(oracle.ristretto_compress(P) for P in pts)
    rc, got, limbs = eng.edwards_vartime_msm(sb, comp, n, want_limbs=True)
    assert rc == 0 and got == want
    point_checks.check_limbs(limbs, want)
    assert eng.edwards_vartime_msm(sb, ext, n, point_fmt=EXTENDED)[:2] == (0, want)
    assert eng.edwards_vartime_msm(dev(sb), dev(comp), n, device_ptrs=True)[:2] == (0, want)
    assert eng.ristretto_vartime_msm(sb, rist, n) == (0, oracle.ristretto_compress(oracle.decompress(want)))
    offs = array.array("Q", [0, n]).tobytes()
    rc, out, ok, limbs = eng.msm_batch(sb, comp, offs, 1, want_limbs=True)
    assert rc == 0 and out == want and ok == b"\x01"
    point_checks.check_limbs(limbs, want)


def test_mostly_even_scalars_single_calls_and_batch(eng, oracle, pool):
    """2000 MSMs of 1..189 terms whose scalars are each even with probability 0.9 (so 43% of full warps are all-even):
    every single call, one msm_batch call over the same segments, and the oracle agree."""
    rnd = random.Random(31337)
    m = 2000
    segs = []
    for _ in range(m):
        n = rnd.randint(1, 189)
        s = [rnd.randrange(pyref.L) for _ in range(n)]
        s = [v & ~1 if rnd.random() < 0.9 else v | 1 for v in s]
        segs.append((s, [rnd.randrange(189) for _ in range(n)]))
    flat_s = b"".join(v.to_bytes(32, "little") for s, _ in segs for v in s)
    flat_p = b"".join(pool["comp"][i] for _, ix in segs for i in ix)
    offs = array.array("Q", [0])
    for s, _ in segs:
        offs.append(offs[-1] + len(s))
    rc, out, ok, _ = eng.msm_batch(flat_s, flat_p, offs.tobytes(), m)
    assert rc == 0 and ok == b"\x01" * m
    bad = []
    for j, (s, ix) in enumerate(segs):
        sb = flat_s[32 * offs[j]:32 * offs[j + 1]]
        want = oracle.compress(oracle.msm("straus_vartime", [v.to_bytes(32, "little") for v in s], [pool["pts"][i] for i in ix]))
        rc, got, _ = eng.edwards_vartime_msm(sb, flat_p[32 * offs[j]:32 * offs[j + 1]], len(s))
        if rc != 0 or got != want or out[32 * j:32 * j + 32] != want:
            bad.append((j, len(s), got == want, out[32 * j:32 * j + 32] == want))
    assert not bad, bad[:10]
