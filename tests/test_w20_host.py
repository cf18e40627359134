"""The limb-parallel (20-lane) field and point code of csrc/warp4_f64.cuh -- w20_sq, w20_invert, w20_add, w20_load / w20_store
and the body of k_combine (Horner pass, encoding, limbs, is_identity) -- executed on the CPU by an emulated warp of 32 host threads
(tests/host/w20_host_check.cpp) with the operand-rule assertions of the host field model switched on, against the
oracle.  CPU only: the emulation is test infrastructure, not a fallback of the product."""
import ctypes as C
import os
import random
import subprocess

import pytest

import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def w20():
    host = os.path.join(ROOT, "tests", "host")
    src = os.path.join(host, "w20_host_check.cpp")
    so = os.path.join(host, "libw20host.so")
    csrc = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
    deps = [src, os.path.join(host, "w4_host_check.cpp")] + [
        os.path.join(csrc, f) for f in ("fe.cuh", "fe64.cuh", "ge.cuh", "ge64.cuh", "warp4_f64.cuh", "straus_vt.cuh", "transcript_warp.cuh", "constants.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src, "-lpthread"])
    lib = C.CDLL(so)
    lib.h_w20_sq_invert.argtypes = [C.c_double * 20]
    return lib


def _points(oracle, rnd, n):
    B = oracle.basepoint()
    return [oracle.scalarmul(rnd.randrange(pyref.L).to_bytes(32, "little"), B) for _ in range(n)]


def _specials(oracle):
    return [oracle.identity(),
            oracle.decompress((pyref.p - 1).to_bytes(32, "little")),       # (0, -1), order 2
            oracle.decompress((0).to_bytes(32, "little"))]                 # order 4


def _limbs_of(v):
    """Balanced radix-2^51 limbs of the integer v < 2^256 (the carry out of the top limb wraps as 19)."""
    out = []
    for _ in range(5):
        l = v & ((1 << 51) - 1)
        if l >= 1 << 50:
            l -= 1 << 51
        out.append(l)
        v = (v - l) >> 51
    out[0] += 19 * v
    return out


def test_20_lane_squaring_and_inversion(w20):
    """w20_sq against fe64_sq and w20_invert (the addition chain of fe_invert) against the integer fe_invert: random
    elements, 0, 1, p - 1, p, 2^255 - 1 as limbs, and limbs at the operand-rule bounds of the squaring (scale < 2, with
    the 2^15 slack) -- every limb at +- the bound, alternating, single non-zero limbs."""
    rnd = random.Random(23)
    B = 1 << 50
    fixed = [_limbs_of(v) for v in (0, 1, pyref.p - 1, pyref.p, 2**255 - 1, 2**255 - 20, 19)]

    def limbs(scale, mode):
        lim = int(scale * B) + (1 << 14)
        if mode == "rand":
            return [rnd.randrange(-lim, lim + 1) for _ in range(5)]
        if mode == "max":
            return [lim] * 5
        if mode == "min":
            return [-lim] * 5
        if mode == "alt":
            return [lim if k % 2 == 0 else -lim for k in range(5)]
        if mode == "one":
            v = [0] * 5; v[rnd.randrange(5)] = rnd.choice((lim, -lim)); return v
        return fixed[rnd.randrange(len(fixed))]

    modes = ("rand", "max", "min", "alt", "one", "fixed")
    cases = [fixed[k:k + 4] for k in range(0, len(fixed), 4)]
    cases[-1] += fixed[:4 - len(cases[-1])]
    for scale in (1.0, 1.5, 1.99):
        for trial in range(24):
            cases.append([limbs(scale, modes[(trial + g) % 6] if trial < 12 else rnd.choice(modes)) for g in range(4)])
    for els in cases:
        a = [float(x) for e in els for x in e]
        assert w20.h_w20_sq_invert((C.c_double * 20)(*a)) == 1, els


def test_20_lane_addition_matches_oracle(w20, oracle):
    """w20_add (the extended addition of w4f_add on 20 lanes): random points, the identity, the order-2 and order-4
    points, P + P and P + (-P)."""
    rnd = random.Random(31)
    pts = _points(oracle, rnd, 4) + _specials(oracle)
    pairs = [(p, q) for p in pts for q in pts]
    pairs += [(p, oracle.sub(oracle.identity(), p)) for p in pts]
    out = (C.c_uint8 * 32)()
    for p, q in pairs:
        assert w20.h_w20_add(out, oracle.compress(p), oracle.compress(q)) == 1
        assert bytes(out) == oracle.compress(oracle.add(p, q))


def _combine(w20, oracle, pts, ranks, nwin, c):
    s = (C.c_uint8 * 32)(); limbs = (C.c_uint64 * 20)(); isid = C.c_uint32()
    rc = w20.h_w20_combine(s, limbs, C.byref(isid), b"".join(oracle.compress(p) for p in pts), ranks, nwin, c)
    assert rc == 1, rc                 # -3: the limb-parallel and the 4-lane forms differ
    return bytes(s), list(limbs), isid.value


@pytest.mark.parametrize("ranks,nwin,c", [(1, 17, 16), (3, 4, 20), (8, 5, 4), (2, 1, 7)])
def test_combine_body_matches_oracle(w20, oracle, ranks, nwin, c):
    """k_combine's body (w20_horner, w20_encode): sum_w 2^(c w) sum_r W[r][w] encoded as the oracle does, limbs of the
    same projective point, is_identity -- and identical outputs to the replicated 4-lane form."""
    rnd = random.Random(ranks * 1000 + nwin + 7)
    pts = _points(oracle, rnd, ranks * nwin)
    sp = _specials(oracle)
    for k in range(min(len(pts), 3)):
        pts[(5 * k + 1) % len(pts)] = sp[k]
    want = oracle.identity()
    for w in range(nwin - 1, -1, -1):
        want = oracle.mul_by_pow_2(want, c) if w != nwin - 1 else want
        for r in range(ranks):
            want = oracle.add(want, pts[r * nwin + w])
    s, limbs, isid = _combine(w20, oracle, pts, ranks, nwin, c)
    assert s == oracle.compress(want)
    assert isid == int(oracle.is_identity(want))
    p = pyref.p
    X, Y, Z, T = (sum(limbs[5 * k + i] << (51 * i) for i in range(5)) for k in range(4))
    wl = oracle.p3_limbs(want)
    Xw, Yw, Zw, Tw = (sum(wl[5 * k + i] << (51 * i) for i in range(5)) for k in range(4))
    assert all(v < p for v in (X, Y, Z, T))                                  # canonical limbs
    assert (X * Zw - Xw * Z) % p == 0 and (Y * Zw - Yw * Z) % p == 0 and (T * Zw - Tw * Z) % p == 0


@pytest.mark.parametrize("ranks,nwin", [(1, 3), (2, 2)])
def test_combine_body_all_identity(w20, oracle, ranks, nwin):
    s, limbs, isid = _combine(w20, oracle, [oracle.identity()] * (ranks * nwin), ranks, nwin, 5)
    assert s == (1).to_bytes(32, "little")
    assert isid == 1
    assert limbs == [0] * 5 + [1, 0, 0, 0, 0] + [1, 0, 0, 0, 0] + [0] * 5


def test_20_lane_store_roundtrip(w20, oracle):
    """w20_store(w20_load(P)): the raw points k_chunk_reduce and k_finish_windows read and write on 20 lanes."""
    rnd = random.Random(47)
    out = (C.c_uint8 * 32)()
    for P in _points(oracle, rnd, 5) + _specials(oracle):
        assert w20.h_w20_store_roundtrip(out, oracle.compress(P)) == 1
        assert bytes(out) == oracle.compress(P)
