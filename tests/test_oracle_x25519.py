"""The X25519 CPU oracle (tests/host/x25519_oracle.c) against the golden vectors, `cryptography` and the Edwards
oracle.  CPU only."""
import json
import os
import random

import pytest

import pyref
import x25519_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def xo():
    return x25519_oracle.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "x25519.json")) as f:
        return json.load(f)


def test_golden_vectors(xo, golden):
    for v in golden["rfc7748_ladder"]:
        assert xo.x25519(bytes.fromhex(v["scalar"]), bytes.fromhex(v["u"])).hex() == v["out"]
    k = u = bytes([9]) + bytes(31)
    want = {v["iterations"]: v["out"] for v in golden["rfc7748_iterated"]}
    for step in range(1, max(want) + 1):
        k, u = xo.x25519(k, u), k
        if step in want:
            assert k.hex() == want[step]
    dh = {n: bytes.fromhex(h) for n, h in golden["rfc7748_dh"].items()}
    assert xo.public_key(dh["alice_private"]) == dh["alice_public"]
    assert xo.public_key(dh["bob_private"]) == dh["bob_public"]
    assert xo.x25519(dh["alice_private"], dh["bob_public"]) == dh["shared"]
    for v in golden["pattern_0x37"]:
        assert xo.public_key(bytes.fromhex(v["scalar"])).hex() == v["out"]
    for h in golden["low_order"] + golden["low_order_bit255"]:
        assert xo.x25519(b"\x5a" * 32, bytes.fromhex(h)) == bytes(32)


def test_clamp_and_mul_bits_be(xo):
    rnd = random.Random(4)
    for _ in range(20):
        k = rnd.randbytes(32)
        c = xo.clamp(k)
        v = int.from_bytes(k, "little")
        assert int.from_bytes(c, "little") == (v & ~7 & (2**255 - 1)) | 2**254
        u = rnd.randbytes(32)
        assert xo.mul_bits_be(u, c, 255) == xo.x25519(k, u)
        assert xo.mul_bits_be(u, c, 256) == xo.x25519(k, u)          # bit 255 of a clamped scalar is 0


def test_matches_cryptography(xo):
    x = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.x25519")
    from cryptography.hazmat.primitives.serialization import Encoding, PublicFormat
    rnd = random.Random(5)
    for _ in range(200):
        k, u = rnd.randbytes(32), rnd.randbytes(32)
        out = xo.x25519(k, u)
        if out != bytes(32):
            assert x.X25519PrivateKey.from_private_bytes(k).exchange(x.X25519PublicKey.from_public_bytes(u)) == out
        pk = x.X25519PrivateKey.from_private_bytes(k).public_key().public_bytes(Encoding.Raw, PublicFormat.Raw)
        assert xo.public_key(k) == pk
    ks, us = rnd.randbytes(32 * 50), rnd.randbytes(32 * 50)
    flat = xo.x25519_batch(ks, us)
    assert flat == b"".join(xo.x25519(ks[32 * i:32 * i + 32], us[32 * i:32 * i + 32]) for i in range(50))


def test_to_montgomery_matches_ladder(xo, oracle):
    """u(clamp(k) B) from the Edwards oracle's point through to_montgomery equals the ladder on u = 9."""
    rnd = random.Random(6)
    B = oracle.basepoint()
    for _ in range(20):
        k = rnd.randbytes(32)
        P = oracle.scalarmul(xo.clamp(k), B)
        P = oracle.add(P, oracle.double(oracle.identity()))                 # Z != 1 after an addition
        assert xo.to_montgomery(oracle.p3_limbs(P)) == xo.public_key(k)
    assert xo.to_montgomery(oracle.p3_limbs(oracle.identity())) == bytes(32)
    # (0, -1) has order 2: u = (1 - 1) / (1 + 1) = 0; the 4-torsion points (+-sqrt(-1), 0) have u = 1
    assert xo.to_montgomery(oracle.p3_limbs(oracle.decompress((pyref.p - 1).to_bytes(32, "little")))) == bytes(32)
    assert xo.to_montgomery(oracle.p3_limbs(oracle.decompress(bytes(32)))) == (1).to_bytes(32, "little")
