"""Host build of the device X25519 ladder (csrc/x25519.cuh) with the fe64 operand-scale assertions on, against the
golden vectors, the X25519 oracle and `cryptography`; and the SASS / resource usage of the ladder kernel in the built
library.  CPU only."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import pytest

import x25519_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curve25519_dalek_b200", "csrc")
LIB = os.path.join(ROOT, "curve25519_dalek_b200", "libdalek_b200.so")
P = 2**255 - 19


@pytest.fixture(scope="module")
def host():
    src = os.path.join(ROOT, "tests", "host", "x25519_host_check.cpp")
    so = os.path.join(ROOT, "tests", "host", "libx25519host.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("x25519.cuh", "fe64.cuh", "fe.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.h_x25519.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    lib.h_x25519_iterate.argtypes = [C.c_void_p, C.c_int]
    lib.h_x25519_iterate.restype = None
    return lib


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "x25519.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def xo():
    return x25519_oracle.load()


def ladder(host, k, u):
    out = (C.c_uint8 * 32)()
    contributory = host.h_x25519(out, bytes(k), bytes(u))
    out = bytes(out)
    assert contributory == (out != bytes(32))
    return out


def b32(x):
    return x.to_bytes(32, "little")


def test_golden_vectors(host, golden):
    for v in golden["rfc7748_ladder"]:
        assert ladder(host, bytes.fromhex(v["scalar"]), bytes.fromhex(v["u"])).hex() == v["out"]
    for v in golden["rfc7748_iterated"]:
        out = (C.c_uint8 * 32)()
        host.h_x25519_iterate(out, v["iterations"])
        assert bytes(out).hex() == v["out"]
    dh = {k: bytes.fromhex(h) for k, h in golden["rfc7748_dh"].items()}
    base = b32(9)
    assert ladder(host, dh["alice_private"], base) == dh["alice_public"]
    assert ladder(host, dh["bob_private"], base) == dh["bob_public"]
    assert ladder(host, dh["alice_private"], dh["bob_public"]) == dh["shared"]
    assert ladder(host, dh["bob_private"], dh["alice_public"]) == dh["shared"]
    for v in golden["pattern_0x37"]:
        assert ladder(host, bytes.fromhex(v["scalar"]), base).hex() == v["out"]


def test_low_order_points_give_zero(host, golden):
    rnd = random.Random(1)
    us = golden["low_order"] + golden["low_order_bit255"]
    assert len(us) == 14
    for h in us:
        for _ in range(3):
            assert ladder(host, rnd.randbytes(32), bytes.fromhex(h)) == bytes(32)


def test_u_and_k_edge_values(host, xo):
    rnd = random.Random(2)
    us = [0, 1, 2, 9, P - 1, P, P + 1, P + 18, 2**255 - 1]
    us += [u | 2**255 for u in us] + [rnd.randrange(2**256) | 2**255 for _ in range(5)]
    ks = [bytes(32), b"\xff" * 32, b"\x37" * 32] + [rnd.randbytes(32) for _ in range(3)]
    for u in us:
        for k in ks:
            assert ladder(host, k, b32(u)) == xo.x25519(k, b32(u)), (k.hex(), hex(u))


def test_random_pairs_match_oracle_and_cryptography(host, xo):
    x25519 = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.x25519")
    rnd = random.Random(3)
    checked = 0
    for i in range(300):
        k = rnd.randbytes(32)
        u = rnd.randbytes(32) if i % 3 else xo.x25519(rnd.randbytes(32), b32(9))   # every third u on the curve
        out = ladder(host, k, u)
        assert out == xo.x25519(k, u)
        if out != bytes(32):                     # cryptography rejects an all-zero shared secret
            got = x25519.X25519PrivateKey.from_private_bytes(k).exchange(x25519.X25519PublicKey.from_public_bytes(u))
            assert got == out
            checked += 1
    assert checked > 250


def _function_sections(text, name):
    """The SASS (or resource line) blocks of every function whose mangled name contains `name`."""
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


def _ladder_kernel():
    return "8k_x25519PK"                         # _Z8k_x25519PKjS0_mPjPh, not k_x25519_base*


def test_ladder_kernel_sass_has_no_indirect_branch():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True)
    blocks = _function_sections(r.stdout, _ladder_kernel())
    assert len(blocks) == 1
    sass = blocks[0]
    assert "DFMA" in sass                        # the FP64 field
    assert not re.search(r"\b(BRX|JMX)\b", sass)


def test_ladder_kernel_does_not_spill():
    if not os.path.exists(LIB):
        pytest.fail("libdalek_b200.so is not built (run __graft_entry__.build())")
    r = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    idx = [i for i, l in enumerate(lines) if re.search(r"Function\s+\S*" + _ladder_kernel(), l)]
    assert len(idx) == 1
    usage = lines[idx[0] + 1]
    assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), usage
