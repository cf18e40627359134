"""The vartime Straus path (csrc/straus_vt.cuh) on the emulated warp of tests/host/w4_host_check.cpp, at scalar patterns
that are uniform across a warp (tests/straus_patterns.py).  Every call checks two things:

  (a) each group's accumulator, as straus_warp_accumulate leaves it before the warp sum: canonical coordinates,
      X Y = Z T, on the curve, and projectively s_j P_j (the identity for a group past n);
  (b) the whole call against the oracle.

A warp whose live scalars are all even ends its loop on digit 0 with no addition anywhere in the warp; the last
doubling must still produce T, since the warp sum reads it.  Most scalars here are short: the loop length does not
change what is being tested, and the emulation costs about one second per 50 digit positions.  CPU only."""
import ctypes as C
import random

import pytest

import point_checks
import straus_patterns as sp
from test_w4_host import w4  # noqa: F401  (the module fixture building the emulation library)


def run(w4, oracle, scalars, points):
    """(a) and (b) for one call of n = len(scalars) terms."""
    n = len(scalars)
    warps = (n + 7) // 8
    groups = (C.c_uint8 * (128 * 8 * max(warps, 1)))()
    out = (C.c_uint8 * 32)()
    enc = b"".join(oracle.compress(P) for P in points)
    rc = w4.h_straus_groups(groups, out, b"".join(v.to_bytes(32, "little") for v in scalars), enc, n)
    assert rc == 1, rc                                             # -1: lanes of a group disagree; -2: a warp sum's T
    raw = bytes(groups)
    for j in range(8 * warps):
        want = sp.scalar_mul_exact(oracle, scalars[j], points[j]) if j < n else oracle.identity()
        point_checks.check_coords(point_checks.coords_from_bytes(raw[128 * j:128 * j + 128]), oracle.compress(want),
                                  what=("group", j, "n", n))
    assert bytes(out) == oracle.compress(sp.msm_exact(oracle, scalars, points)), n


@pytest.mark.parametrize("n", range(1, 17))
def test_all_even_warps(w4, oracle, n):
    """1..8 live groups per warp, one and two warps, every scalar even.  Before the last doubling refreshed T, n = 5..8
    gave a wrong sum and every n gave stale group accumulators."""
    rnd = random.Random(100 + n)
    bits = 253 if n in (5, 8, 16) else 24
    run(w4, oracle, sp.layout(n, {}, "even", rnd, bits), sp.random_points(oracle, rnd, n))


@pytest.mark.parametrize("k", sp.K_TRAILING)
def test_trailing_zero_digits_shared_by_the_warp(w4, oracle, k):
    """Every scalar a multiple of 2^k: the last k digit positions only double."""
    rnd = random.Random(200 + k)
    for n in (5, 8) if k >= 200 else (7,):
        run(w4, oracle, sp.layout(n, {}, "pow2_%d" % k, rnd, 253 if k >= 200 else 24 + k), sp.random_points(oracle, rnd, n))


def test_one_odd_scalar_in_each_position(w4, oracle):
    """Control: one odd scalar among even ones makes the warp add at digit 0, in each of the eight positions."""
    rnd = random.Random(300)
    pts = sp.random_points(oracle, rnd, 8)
    for i in range(8):
        run(w4, oracle, sp.pattern_scalars("odd_at_%d" % i, rnd, 8, 24), pts)


@pytest.mark.parametrize("pattern", ["ones", "small_odd"])
def test_no_doubling_at_all(w4, oracle, pattern):
    """Every top digit is digit 0: the loop runs once, adds, and never doubles."""
    rnd = random.Random(400)
    for n in (1, 5, 8, 13):
        run(w4, oracle, sp.layout(n, {}, pattern, rnd), sp.random_points(oracle, rnd, n))


def test_zero_warp_between_live_warps(w4, oracle):
    """Warp 1 of 3 has only zero scalars (it never enters its loop); warps 0 and 2 are all-even."""
    rnd = random.Random(500)
    n = 21
    run(w4, oracle, sp.layout(n, {1: "zero"}, "even", rnd, 24), sp.random_points(oracle, rnd, n))


def test_even_scalars_with_bit_255(w4, oracle):
    """Even scalars beyond the reference's Scalar invariant, one of them 2^256 - 2: the NAF runs past digit 255."""
    rnd = random.Random(600)
    run(w4, oracle, sp.pattern_scalars("even_bit255", rnd, 6), sp.random_points(oracle, rnd, 6))


def test_identity_and_small_order_points_in_an_all_even_warp(w4, oracle):
    rnd = random.Random(700)
    pts = sp.small_order_points(oracle) + sp.random_points(oracle, rnd, 3)
    rnd.shuffle(pts)
    run(w4, oracle, sp.pattern_scalars("even", rnd, 7, 24), pts)


def test_recorded_benchmark_warps(w4, oracle):
    """The all-even warp of each of the two inputs on which the single vartime call once disagreed with the oracle
    (tests/golden/straus_all_even_warps.json: 16384x64 sample 24 warp 3, ragged_8192 sample 41 warp 13), 8 terms each."""
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "straus_all_even_warps.json")) as f:
        cases = json.load(f)["cases"]
    for c in cases:
        w = c["all_even_warp"]
        s = [int.from_bytes(bytes.fromhex(x), "little") for x in c["scalars"][8 * w:8 * w + 8]]
        assert all(v % 2 == 0 for v in s)
        pts = [oracle.decompress(bytes.fromhex(x)) for x in c["points"][8 * w:8 * w + 8]]
        run(w4, oracle, s, pts)
