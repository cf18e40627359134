"""Scalar patterns that are uniform across a warp of the vartime Straus path, and an exact reference for them.

The Straus path (csrc/straus_vt.cuh) runs one warp per eight terms: term j is group j % 8 of warp j // 8, and every
decision of the main loop (where it starts, whether a digit position adds at all) is taken per warp.  Random scalars
almost never make such a decision the same for all eight groups -- all eight scalars even, say, happens once in 256
warps -- so these generators make it so on purpose: every live scalar of a warp even, a multiple of 2^k, odd and
small (no doubling at all), or zero."""
import random

import pyref

L = pyref.L
K_TRAILING = (2, 5, 6, 64, 200, 250)


def _even(rnd, bits):
    return rnd.randrange(1, 1 << (bits - 1)) << 1


def pattern_scalars(pattern, rnd, count, bits=253):
    """count scalars (ints) of one warp following `pattern`; bits bounds the size of the random part.
      even            every scalar even and non-zero
      pow2_<k>        every scalar a non-zero multiple of 2^k: k trailing doublings with no addition
      odd_at_<i>      every scalar even except the one at index i (the control of `even`)
      ones            every scalar 1: the top digit is digit 0, no doubling at all
      small_odd       odd scalars below 16: one digit each, digit 0
      zero            every scalar 0
      even_bit255     even scalars with bit 255 set (legal at the engine's boundary), the last one 2^256 - 2"""
    if pattern == "even":
        return [_even(rnd, bits) for _ in range(count)]
    if pattern.startswith("pow2_"):
        k = int(pattern[5:])
        top = max(bits, k + 3)
        return [rnd.randrange(1, 1 << (top - k)) << k for _ in range(count)]
    if pattern.startswith("odd_at_"):
        i = int(pattern[7:])
        s = [_even(rnd, bits) for _ in range(count)]
        if i < count:
            s[i] |= 1
        return s
    if pattern == "ones":
        return [1] * count
    if pattern == "small_odd":
        return [rnd.randrange(1, 16, 2) for _ in range(count)]
    if pattern == "zero":
        return [0] * count
    if pattern == "even_bit255":
        s = [(1 << 255) | _even(rnd, min(bits, 255)) for _ in range(count)]
        s[-1] = (1 << 256) - 2
        return s
    raise ValueError(pattern)


def layout(n, warp_patterns, default, rnd, bits=253):
    """n scalars: warp w follows warp_patterns.get(w, default)."""
    out = []
    for w in range((n + 7) // 8):
        cnt = min(8, n - 8 * w)
        out += pattern_scalars(warp_patterns.get(w, default), rnd, cnt, bits)
    return out


def scalar_mul_exact(oracle, v, P):
    """v * P for any 256-bit integer v (the oracle's scalar multiplication takes v < 2^252 here): v = lo + 2^252 hi."""
    lo = oracle.scalarmul((v % (1 << 252)).to_bytes(32, "little"), P)
    if v >> 252 == 0:
        return lo
    hi = oracle.mul_by_pow_2(oracle.scalarmul((v >> 252).to_bytes(32, "little"), P), 252)
    return oracle.add(lo, hi)


def msm_exact(oracle, scalars, points):
    """sum s_i P_i for integer scalars: the oracle's vartime Straus (straus.rs:159-200) when every scalar has bit 255
    clear (the reference's Scalar invariant), exact integer arithmetic otherwise."""
    if all(v < 1 << 255 for v in scalars):
        return oracle.msm("straus_vartime", [v.to_bytes(32, "little") for v in scalars], points)
    acc = oracle.identity()
    for v, P in zip(scalars, points):
        acc = oracle.add(acc, scalar_mul_exact(oracle, v, P))
    return acc


def random_points(oracle, rnd, n):
    B = oracle.basepoint()
    return [oracle.scalarmul(rnd.randrange(L).to_bytes(32, "little"), B) for _ in range(n)]


def small_order_points(oracle):
    """identity, (0, -1) of order 2, (x, 0) of order 4 and an order-8 point."""
    return [oracle.identity(), oracle.decompress((pyref.p - 1).to_bytes(32, "little")),
            oracle.decompress((0).to_bytes(32, "little")),
            oracle.decompress(bytes.fromhex("26e8958fc2b227b045c3f489f2ef98f0d5dfac05d3c63339b13802886d53fc05"))]
