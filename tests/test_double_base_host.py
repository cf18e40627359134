"""Host build of the device double-base scalar multiplication a P + b B (csrc/double_base.cuh) with the fe64
operand-scale and limb-bound assertions on, against the C oracles; the faithful NAF oracle of vartime_double_base.rs
against the oracle library's Straus value and pyref; and the resource usage of the double-base kernels and of the
Ed25519 verifier that shares the device routine.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

import double_base_oracle as dbo_mod
import oracle_lib
import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
L = pyref.L
PRIME = 2**255 - 19
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2


@pytest.fixture(scope="module")
def host():
    src = os.path.join(ROOT, "tests", "host", "double_base_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libdoublebasehost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("double_base.cuh", "ge64.cuh", "ge.cuh", "fe64.cuh", "fe.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_double_base.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int]
    return lib


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def dbo():
    return dbo_mod.load()


@pytest.fixture(scope="module")
def torsion():
    with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json")) as f:
        return json.load(f)["EIGHT_TORSION"]


def dbl(host, a, point, b, fmt=COMPRESSED):
    out = (C.c_uint8 * 32)()
    ok = host.h_double_base(out, bytes(a) + bytes(b), bytes(point), fmt)
    return bytes(out), ok


def b32(x):
    return x.to_bytes(32, "little")


def limbs_bytes(limbs):
    return b"".join(int(v).to_bytes(8, "little") for v in limbs)


def edge_scalars():
    """0, 1, l - 1, l, l + 1, 2^255 - 1, 2^252 and the radix-16 carry patterns"""
    return [b32(0), b32(1), b32(L - 1), b32(L), b32(L + 1), b32(2**255 - 1), b32(2**252), bytes([0x88] * 31 + [0x08]),
            bytes([0x88] * 31 + [0x78]), bytes([0x77] * 32), bytes([0xff] * 31 + [0x0f]), bytes([0xff] * 31 + [0x7f]),
            bytes([0x08] * 32), bytes([0xf8] * 31 + [0x7f])]


def want(orc, a, P, b):
    """a P + b B by the oracle library's scalar multiplication and addition (independent of both double-base paths)"""
    return orc.add(orc.scalarmul(a, P), orc.scalarmul(b, orc.basepoint()))


def test_kat(host, dbo):
    with open(os.path.join(ROOT, "tests", "golden", "kat.json")) as f:
        ek = json.load(f)["edwards"]
    a, b = bytes.fromhex(ek["A_SCALAR"]["hex"]), bytes.fromhex(ek["B_SCALAR"]["hex"])
    A = bytes.fromhex(ek["A_TIMES_BASEPOINT"]["hex"])
    res = bytes.fromhex(ek["DOUBLE_SCALAR_MULT_RESULT"]["hex"])
    assert dbl(host, a, A, b) == (res, 1)
    assert dbo.one(a, A, b) == (res, 1)
    assert dbo.one(a, A, b, naf=False) == (res, 1)


def test_edge_scalars_for_a_and_b(host, dbo, orc):
    rnd = random.Random(21)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    enc = orc.compress(P)
    r = b32(rnd.randrange(L))
    for s in edge_scalars():
        assert s[31] < 128
        for a, b in ((s, r), (r, s), (s, s)):
            got = dbl(host, a, enc, b)
            assert got == dbo.one(a, enc, b), (a.hex(), b.hex())
            assert got[0] == orc.compress(want(orc, a, P, b))


def test_special_points(host, dbo, orc, torsion):
    rnd = random.Random(22)
    B = orc.basepoint()
    pts = [orc.identity(), B] + [orc.p3_from_limbs(t["limbs"]) for t in torsion]
    pts += [orc.add(orc.scalarmul(b32(rnd.randrange(L)), B), orc.p3_from_limbs(t["limbs"])) for t in torsion]
    pts += [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(4)]
    for P in pts:
        enc = orc.compress(P)
        for a, b in [(s, b32(rnd.randrange(L))) for s in edge_scalars()[:6]] + [(b32(rnd.randrange(2**255)), b32(rnd.randrange(2**255)))]:
            got = dbl(host, a, enc, b)
            assert got == dbo.one(a, enc, b)
            assert got[0] == orc.compress(want(orc, a, P, b))


def test_unreduced_scalars_on_torsion_points(host, dbo, orc, torsion):
    """a in [l, 2^255) is used as given: on a point with a torsion component a A != (a mod l) A"""
    rnd = random.Random(23)
    B = orc.basepoint()
    hits = 0
    for t in torsion[1:]:
        P = orc.add(orc.scalarmul(b32(rnd.randrange(1, L)), B), orc.p3_from_limbs(t["limbs"]))
        enc = orc.compress(P)
        for a_int in (L, L + 1, L + 3, 2**255 - 1, rnd.randrange(L, 2**255)):
            a, b = b32(a_int), b32(rnd.randrange(2**255))
            got = dbl(host, a, enc, b)
            reduced = dbo.one(b32(a_int % L), enc, b)
            assert got == dbo.one(a, enc, b)
            if reduced != got:
                hits += 1
    assert hits >= 20                                  # the case has teeth: most of the 35 differ from the reduced value


def test_extended_input_with_any_z(host, orc):
    rnd = random.Random(24)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    x, y = [int.from_bytes(orc.fe_to_bytes(c), "little") for c in (P.X, P.Y)]
    zi = pow(int.from_bytes(orc.fe_to_bytes(P.Z), "little"), PRIME - 2, PRIME)
    x, y = x * zi % PRIME, y * zi % PRIME
    for lam in [1, 2, PRIME - 1, rnd.randrange(1, PRIME)]:
        coords = [lam * x % PRIME, lam * y % PRIME, lam, lam * x * y % PRIME]
        limbs = [(c >> (51 * k)) & (2**51 - 1) for c in coords for k in range(5)]
        a, b = b32(rnd.randrange(2**255)), b32(rnd.randrange(L))
        assert dbl(host, a, limbs_bytes(limbs), b, EXTENDED) == (orc.compress(want(orc, a, P, b)), 1)


def test_ristretto(host, dbo, orc):
    rnd = random.Random(25)
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        classes = json.load(f)["classes"]
    for _ in range(8):
        enc = orc.ristretto_compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint()))
        a, b = b32(rnd.randrange(2**255)), b32(rnd.randrange(2**255))
        got = dbl(host, a, enc, b, RISTRETTO)
        assert got == dbo.one(a, enc, b, RISTRETTO)
        assert got == (orc.ristretto_compress(want(orc, a, orc.ristretto_decompress(enc), b)), 1)
    for cls in ("noncanonical", "negative", "nonsquare", "t_negative", "y_zero"):
        for v in classes[cls]:
            assert dbl(host, b32(5), bytes.fromhex(v["s"]), b32(9), RISTRETTO) == (bytes(32), 0), (cls, v["s"])
            assert dbo.one(b32(5), bytes.fromhex(v["s"]), b32(9), RISTRETTO) == (bytes(32), 0)


def test_undecodable_edwards_point(host, dbo):
    # y = 2 is not the y of a curve point
    assert dbl(host, b32(7), b32(2), b32(3)) == (b32(1), 0)
    assert dbo.one(b32(7), b32(2), b32(3)) == (b32(1), 0)


def test_naf_oracle_matches_straus_and_pyref(dbo, orc):
    """the line-faithful restatement of vartime_double_base.rs against the oracle library's Straus value (300 inputs)
    and pyref's big-integer arithmetic (the first 60)"""
    rnd = random.Random(26)
    Bp = pyref.B
    for i in range(300):
        t = rnd.randrange(1, L)
        a = b32(rnd.randrange(2**255) if i % 3 else rnd.randrange(L))
        b = b32(rnd.randrange(2**255) if i % 2 else rnd.randrange(L))
        if i % 50 == 0:
            a = b32(0)
        enc = orc.compress(orc.scalarmul(b32(t), orc.basepoint()))
        got = dbo.one(a, enc, b)
        assert got == dbo.one(a, enc, b, naf=False), i
        if i < 60:
            A = pyref.mul(t, Bp)
            assert got[0] == pyref.compress(pyref.add(pyref.mul(pyref.sc(a), A), pyref.mul(pyref.sc(b), Bp))), i


def test_oracle_batch_matches_items(dbo, orc):
    rnd = random.Random(27)
    n = 37
    ab = [b32(rnd.randrange(2**255)) + b32(rnd.randrange(2**255)) for _ in range(n)]
    pts = [orc.compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())) for _ in range(n)]
    pts[5] = b32(2)
    for threads in (1, 4):
        rc, out, ok = dbo.batch(b"".join(ab), b"".join(pts), n, COMPRESSED, threads)
        assert rc == 1 and ok == bytes(1 if i != 5 else 0 for i in range(n))
        assert [out[32 * i:32 * i + 32] for i in range(n)] == [dbo.one(x[:32], p, x[32:])[0] for x, p in zip(ab, pts)]


def _res_usage():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    out = {}
    for i, l in enumerate(lines):
        m = re.search(r"Function\s+(\S+):", l)
        if m:
            u = dict(re.findall(r"(REG|STACK|LOCAL):(\d+)", lines[i + 1]))
            out[m.group(1)] = {k: int(v) for k, v in u.items()}
    return out


# ptxas figures of the sm_90a build (nvcc 12.9, -O3): the double-base kernels, and the Ed25519 verifier kernels whose
# evaluation loop moved into double_base.cuh unchanged (the same figures as before the move)
DOUBLE_BASE_USAGE = {"REG": 252, "STACK": 1472, "LOCAL": 0}
VERIFY_EACH_USAGE = {"REG": 252, "STACK": 1472, "LOCAL": 0}


def test_double_base_kernels_resource_usage():
    usage = _res_usage()
    kernels = {k: v for k, v in usage.items() if "21k_vartime_double_baseILi" in k}
    assert len(kernels) == 3, sorted(kernels)
    for k, v in kernels.items():
        print(k, v)
        assert v == DOUBLE_BASE_USAGE, k


def test_verify_each_resource_usage_unchanged():
    usage = _res_usage()
    kernels = {k: v for k, v in usage.items() if re.match(r"_Z1[36]k_verify_each(_ph)?P", k)}
    assert len(kernels) == 2, sorted(kernels)
    for k, v in kernels.items():
        assert v == VERIFY_EACH_USAGE, k


def test_double_base_kernels_sass():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    blocks, cur = [], None
    for line in r.stdout.splitlines():
        m = re.search(r"Function\s*:\s*(\S+)", line)
        if m:
            cur = [] if "21k_vartime_double_baseILi" in m.group(1) else None
            if cur is not None:
                blocks.append(cur)
        if cur is not None:
            cur.append(line)
    assert len(blocks) == 3
    for b in blocks:
        assert "DFMA" in "\n".join(b)                  # the FP64 field
