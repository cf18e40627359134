"""MontgomeryPoint on the CPU: the oracle (tests/host/montgomery_oracle.c) against the reference's own unit tests and an
independent big-integer ladder; the host build of the generalised device ladder (mont_ladder<NW> in csrc/x25519.cuh)
with the fe64 operand-scale assertions on, against the oracle, for every bit length the kernels special-case and edge u
values; and the SASS / resource usage of the new kernels in the built library.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

import montgomery_oracle
import pyref
import x25519_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
P = 2**255 - 19
NBITS = [0, 1, 2, 254, 255, 256, 511, 512]


@pytest.fixture(scope="module")
def mo():
    return montgomery_oracle.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "x25519.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def host():
    src = os.path.join(ROOT, "tests", "host", "montgomery_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libmontgomeryhost.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("x25519.cuh", "fe64.cuh", "fe.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_mont_ladder.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_char_p]
    lib.h_mont_ladder.restype = None
    return lib


def b32(x):
    return x.to_bytes(32, "little")


def host_ladder(host, ints, nbits, u):
    out = (C.c_uint8 * 32)()
    host.h_mont_ladder(out, bytes(ints), len(ints), nbits, bytes(u))
    return bytes(out)


def py_ladder(u_bytes, b, nbits):
    """Costello-Smith algorithm 8 on Python integers (montgomery.rs:176-211, :430-468), independent of both C sources."""
    u = int.from_bytes(u_bytes, "little") & (2**255 - 1)
    x0, x1 = (1, 0), (u % P, 1)
    prev = 0
    for i in range(nbits - 1, -1, -1):
        bit = (b >> i) & 1
        if prev ^ bit:
            x0, x1 = x1, x0
        (U0, W0), (U1, W1) = x0, x1
        t4, t5 = (U0 + W0) ** 2 % P, (U0 - W0) ** 2 % P
        t6 = (t4 - t5) % P
        t9, t10 = ((U0 + W0) * (U1 - W1) + (U0 - W0) * (U1 + W1)) % P, ((U0 + W0) * (U1 - W1) - (U0 - W0) * (U1 + W1)) % P
        x0 = (t4 * t5 % P, t6 * (121666 * t6 + t5) % P)
        x1 = (t9 * t9 % P, u * t10 * t10 % P)
        prev = bit
    if prev:
        x0, x1 = x1, x0
    U, W = x0
    return b32(U * pow(W, P - 2, P) % P)


def edge_us(golden):
    us = [b32(x) for x in (0, 1, 9, P - 1, P, P + 1, 2**255 - 1)]
    us += [b32(int.from_bytes(u, "little") | 2**255) for u in us]          # the bit-255 twins
    us += [bytes.fromhex(h) for h in golden["low_order"] + golden["low_order_bit255"]]
    return us


# ---- the oracle against the reference's unit tests (montgomery.rs:556-613) ----

def test_oracle_basepoint_montgomery_to_edwards(mo):
    B = pyref.compress(pyref.B)
    minus_B = pyref.compress(pyref.neg(pyref.B))
    assert mo.to_edwards(b32(9), 0) == B
    assert mo.to_edwards(b32(9), 1) == minus_B
    assert mo.to_edwards(b32(9), 2) == B                       # sign << 7 on a u8: only bit 0 counts
    assert mo.to_edwards(b32(9), 0xff) == minus_B


def test_oracle_montgomery_to_edwards_rejects_twist(mo):
    assert mo.to_edwards(b32(2), 0) is None
    assert mo.to_edwards(b32(P - 1), 0) is None
    assert mo.to_edwards(b32(P - 1), 1) is None
    assert mo.to_edwards(b32((P - 1) | 2**255), 0) is None      # the other encoding of -1


def test_oracle_eq_defined_mod_p(mo):
    u18, u18_unred = b32(18), b"\xff" * 32
    rnd = random.Random(1)
    for nbits in (255, 512):
        b = rnd.randbytes(64)
        assert mo.mul_bits_be(u18, b, nbits) == mo.mul_bits_be(u18_unred, b, nbits)
    assert mo.to_edwards(u18, 0) == mo.to_edwards(u18_unred, 0)
    assert mo.to_edwards(u18, 1) == mo.to_edwards(u18_unred, 1)


def test_oracle_u0_gives_the_order_two_point(mo):
    minus_one_y = b32(P - 1)                                  # (0, -1): x = 0 compresses with sign 0
    assert mo.to_edwards(b32(0), 0) == minus_one_y
    assert mo.to_edwards(b32(0), 1) == minus_one_y


def test_oracle_to_edwards_round_trips_edwards_points(mo):
    rnd = random.Random(2)
    for _ in range(20):
        Pt = pyref.mul(rnd.randrange(pyref.L), pyref.B)
        x, y = Pt
        u = (1 + y) * pyref.inv(1 - y) % P
        assert mo.to_edwards(b32(u), x & 1) == pyref.compress(Pt)


def test_oracle_ladder_matches_python_and_x25519(mo):
    rnd = random.Random(3)
    xo = x25519_oracle.load()
    for nbits in NBITS:
        for _ in range(3):
            b = rnd.randbytes(64)
            u = rnd.randbytes(32)
            assert mo.mul_bits_be(u, b, nbits) == py_ladder(u, int.from_bytes(b, "little"), nbits), nbits
    for _ in range(10):
        k, u = rnd.randbytes(32), rnd.randbytes(32)
        assert mo.mul_bits_be(u, xo.clamp(k), 255) == xo.x25519(k, u)


def test_oracle_mul_base_formats(mo):
    rnd = random.Random(4)
    xo = x25519_oracle.load()
    for _ in range(5):
        s = rnd.randrange(2**255)
        Pt = pyref.mul(s, pyref.B)
        assert mo.mul_base(b32(s), montgomery_oracle.FMT_COMPRESSED) == pyref.compress(Pt)
        assert mo.mul_base(b32(s), montgomery_oracle.FMT_MONTGOMERY) == mo.mul(b32(s % pyref.L), b32(9))
        k = rnd.randbytes(32)
        assert mo.mul_base(k, montgomery_oracle.FMT_MONTGOMERY, clamp=True) == xo.public_key(k)
    assert mo.mul_base(bytes(32), montgomery_oracle.FMT_MONTGOMERY) == bytes(32)          # the identity: u = 0


# ---- the host-compiled device ladder against the oracle ----

@pytest.mark.parametrize("nbits", NBITS)
def test_host_ladder_edge_u(host, mo, golden, nbits):
    rnd = random.Random(10 + nbits)
    nbytes = max(1, (nbits + 7) // 8)
    ints = [bytes(nbytes), b"\xff" * nbytes, rnd.randbytes(nbytes), rnd.randbytes(64)]
    for u in edge_us(golden):
        for b in ints:
            if nbits > 8 * len(b):
                continue
            assert host_ladder(host, b, nbits, u) == mo.mul_bits_be(u, b, nbits), (nbits, b.hex(), u.hex())


@pytest.mark.parametrize("nbits", NBITS)
def test_host_ladder_random(host, mo, nbits):
    rnd = random.Random(20 + nbits)
    for int_bytes in sorted({1, 32, 33, 64, max(1, (nbits + 7) // 8)}):
        if nbits > 8 * int_bytes:
            continue
        for _ in range(4):
            b, u = rnd.randbytes(int_bytes), rnd.randbytes(32)
            assert host_ladder(host, b, nbits, u) == mo.mul_bits_be(u, b, nbits), (nbits, int_bytes)


def test_host_ladder_low_order_points_give_zero(host, golden):
    rnd = random.Random(5)
    for h in golden["low_order"] + golden["low_order_bit255"]:
        b = rnd.randbytes(32)
        b = b[:-1] + bytes([b[-1] & 0x7f])
        b = bytes([b[0] & 0xf8]) + b[1:]                       # a multiple of 8: every low-order point goes to u = 0
        assert host_ladder(host, b, 255, bytes.fromhex(h)) == bytes(32)


# ---- SASS and resources of the new kernels ----

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


NEW_KERNELS = {"13k_mont_ladder": 2, "17k_mont_to_edwards": 1, "13k_x25519_base": 5}
LADDER_KERNELS = ["13k_mont_ladder"]


def _lib_or_fail():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")


def test_new_kernels_sass_have_no_indirect_branch():
    _lib_or_fail()
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    for name, count in NEW_KERNELS.items():
        blocks = _function_sections(r.stdout, name)
        assert len(blocks) == count, name
        for sass in blocks:
            assert "DFMA" in sass                               # the FP64 field
            assert not re.search(r"\b(BRX|JMX)\b", sass), name


def test_ladder_kernels_do_not_spill():
    _lib_or_fail()
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    for name in LADDER_KERNELS:
        idx = [i for i, l in enumerate(lines) if re.search(r"Function\s+\S*" + name, l)]
        assert len(idx) == 2, name                              # the 8- and 16-word instances
        for i in idx:
            usage = lines[i + 1]
            assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), (lines[i], usage)
