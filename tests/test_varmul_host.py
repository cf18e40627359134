"""Host build of the device variable-base scalar multiplication (csrc/varmul.cuh) with the fe64 operand-scale assertions
on, against the golden vectors of tests/golden/scalar_mul.json and the C oracle; and the SASS / resource usage of the
new kernels in the built library.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

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
    src = os.path.join(ROOT, "tests", "host", "varmul_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libvarmulhost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("varmul.cuh", "x25519.cuh", "ge64.cuh", "ge.cuh", "fe64.cuh", "fe.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_mul.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    lib.h_torsion.argtypes = [C.c_char_p, C.c_int]
    return lib


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json")) as f:
        return json.load(f)


def mul(host, s, point, fmt=COMPRESSED, clamp=False):
    out = (C.c_uint8 * 32)()
    ok = host.h_mul(out, bytes(s), bytes(point), fmt, 1 if clamp else 0)
    return bytes(out), ok


def clamp(b):
    b = bytearray(b)
    b[0] &= 248
    b[31] &= 127
    b[31] |= 64
    return bytes(b)


def b32(x):
    return x.to_bytes(32, "little")


def limbs_bytes(limbs):
    return b"".join(int(v).to_bytes(8, "little") for v in limbs)


def edge_scalars():
    return [b32(0), b32(1), b32(L - 1), b32(L), b32(L + 1), b32(2**255 - 1), b32(2**252), bytes([0x88] * 31 + [0x08]),
            bytes([0x88] * 31 + [0x78]), bytes([0x77] * 32), bytes([0xff] * 31 + [0x0f]), bytes([0xff] * 31 + [0x7f]),
            bytes([0x08] * 32), bytes([0xf8] * 31 + [0x7f])]


def test_golden_vectors(host, golden):
    a, base = bytes.fromhex(golden["A_SCALAR"]), bytes.fromhex(golden["BASEPOINT"])
    aB = bytes.fromhex(golden["A_TIMES_BASEPOINT"])
    assert mul(host, a, base) == (aB, 1)
    assert mul(host, a, aB)[0].hex() == golden["A_TIMES_A_TIMES_BASEPOINT"]
    assert mul(host, bytes.fromhex(golden["BASEPOINT_ORDER"]), base)[0].hex() == golden["IDENTITY"]
    for t in golden["EIGHT_TORSION"]:
        assert mul(host, b32(1), bytes.fromhex(t["compressed"]))[0].hex() == t["compressed"]
        assert mul(host, b32(8), bytes.fromhex(t["compressed"]))[0].hex() == golden["IDENTITY"]


def test_random_points_and_scalars(host, orc):
    rnd = random.Random(11)
    B = orc.basepoint()
    for i in range(60):
        P = orc.scalarmul(b32(rnd.randrange(L)), B)
        s = b32(rnd.randrange(2**255)) if i % 2 else b32(rnd.randrange(L))
        assert mul(host, s, orc.compress(P)) == (orc.compress(orc.scalarmul(s, P)), 1)


def test_edge_scalars(host, orc):
    rnd = random.Random(12)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    enc = orc.compress(P)
    for s in edge_scalars():
        assert s[31] < 128
        assert mul(host, s, enc)[0] == orc.compress(orc.scalarmul(s, P)), s.hex()


def test_clamped_scalars(host, orc):
    rnd = random.Random(13)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    enc = orc.compress(P)
    for s in [b"\xff" * 32, bytes(32), b"\x80" * 32] + [rnd.randbytes(32) for _ in range(10)]:
        assert mul(host, s, enc, clamp=True)[0] == orc.compress(orc.scalarmul(clamp(s), P)), s.hex()


def test_identity_torsion_and_mixed_points(host, orc, golden):
    rnd = random.Random(14)
    B = orc.basepoint()
    pts = [orc.identity()] + [orc.p3_from_limbs(t["limbs"]) for t in golden["EIGHT_TORSION"]]
    pts += [orc.add(orc.scalarmul(b32(rnd.randrange(L)), B), orc.p3_from_limbs(t["limbs"])) for t in golden["EIGHT_TORSION"]]
    for P in pts:
        enc = orc.compress(P)
        for s in edge_scalars()[:6] + [b32(rnd.randrange(L)) for _ in range(2)]:
            assert mul(host, s, enc)[0] == orc.compress(orc.scalarmul(s, P))


def test_extended_input_with_any_z(host, orc):
    rnd = random.Random(15)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    x, y = [int.from_bytes(orc.fe_to_bytes(c), "little") for c in (P.X, P.Y)]
    z0 = int.from_bytes(orc.fe_to_bytes(P.Z), "little")
    zi = pow(z0, PRIME - 2, PRIME)
    x, y = x * zi % PRIME, y * zi % PRIME
    for lam in [1, 2, PRIME - 1, rnd.randrange(1, PRIME)]:
        coords = [lam * x % PRIME, lam * y % PRIME, lam, lam * x * y % PRIME]
        limbs = [(c >> (51 * k)) & (2**51 - 1) for c in coords for k in range(5)]
        s = b32(rnd.randrange(L))
        assert mul(host, s, limbs_bytes(limbs), EXTENDED) == (orc.compress(orc.scalarmul(s, P)), 1)


def test_ristretto(host, orc):
    rnd = random.Random(16)
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        rist = json.load(f)
    encs = [orc.ristretto_compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())) for _ in range(12)]
    for enc in encs:
        for s in edge_scalars()[:6] + [b32(rnd.randrange(L))]:
            want = orc.ristretto_compress(orc.scalarmul(s, orc.ristretto_decompress(enc)))
            assert mul(host, s, enc, RISTRETTO) == (want, 1)
    classes = rist["classes"]
    for cls in ("noncanonical", "negative", "nonsquare", "t_negative", "y_zero"):
        for v in classes[cls]:
            assert mul(host, b32(5), bytes.fromhex(v["s"]), RISTRETTO) == (bytes(32), 0), (cls, v["s"])
    for v in classes["valid"]:
        enc = bytes.fromhex(v["s"])
        want = orc.ristretto_compress(orc.scalarmul(b32(5), orc.ristretto_decompress(enc)))
        assert mul(host, b32(5), enc, RISTRETTO) == (want, 1)


def test_undecodable_edwards_point(host):
    # y = 2 is not the y of a curve point
    assert mul(host, b32(7), b32(2)) == (b32(1), 0)


def test_torsion_flags(host, orc, golden):
    rnd = random.Random(17)
    B = orc.basepoint()
    for t in golden["EIGHT_TORSION"]:
        want = 1 | (2 if t["compressed"] == golden["IDENTITY"] else 0) | 4
        assert host.h_torsion(bytes.fromhex(t["compressed"]), COMPRESSED) == want
        assert host.h_torsion(limbs_bytes(t["limbs"]), EXTENDED) == want
    for _ in range(6):
        P = orc.scalarmul(b32(rnd.randrange(1, L)), B)
        assert host.h_torsion(orc.compress(P), COMPRESSED) == 2 | 4
        T = orc.p3_from_limbs(golden["EIGHT_TORSION"][rnd.randrange(1, 8)]["limbs"])
        assert host.h_torsion(orc.compress(orc.add(P, T)), COMPRESSED) == 4
    assert host.h_torsion(b32(2), COMPRESSED) == 0


def _function_sections(text, name):
    blocks, cur = [], None
    for line in text.splitlines():
        m = re.search(r"Function\s*:\s*(\S+)", line)
        if m:
            cur = [] if name in m.group(1) else None
            if cur is not None:
                blocks.append(cur)
        if cur is not None:
            cur.append(line)
    return ["\n".join(b) for b in blocks]


KERNELS = ["8k_varmulILi", "13k_varmul_combILi", "9k_torsionILi"]


def test_kernels_sass_has_no_indirect_branch():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    for k in KERNELS:
        blocks = _function_sections(r.stdout, k)
        assert len(blocks) == (2 if k.startswith("9k_torsion") else 3), k
        for sass in blocks:
            assert "DFMA" in sass                    # the FP64 field
            assert not re.search(r"\b(BRX|JMX)\b", sass)


def test_kernels_resource_usage():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    found = 0
    for i, l in enumerate(lines):
        if any(re.search(r"Function\s+\S*" + k, l) for k in KERNELS):
            print(l.strip(), lines[i + 1].strip())
            assert re.search(r"REG:\d+", lines[i + 1])
            found += 1
    assert found == 8


@pytest.mark.parametrize("pattern", ["even", "pow2_2", "pow2_5", "pow2_6", "pow2_64", "pow2_200", "pow2_250"])
def test_scalars_with_trailing_zero_bits(host, orc, pattern):
    """Even scalars and multiples of 2^k end on doublings with no addition: the result must still carry T = XY / Z
    (h_mul returns -2 otherwise)."""
    import straus_patterns as sp
    rnd = random.Random(pattern)
    P = orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())
    for s in sp.pattern_scalars(pattern, rnd, 6):
        assert mul(host, b32(s), orc.compress(P)) == (orc.compress(orc.scalarmul(b32(s), P)), 1), hex(s)
