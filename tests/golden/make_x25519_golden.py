"""Writes tests/golden/x25519.json: the X25519 known-answer vectors of the tests.

  rfc7748_ladder      RFC 7748 section 5.2, the two (scalar, u) -> output vectors
  rfc7748_iterated    RFC 7748 section 5.2, k = u = 9 iterated (k, u) <- (x25519(k, u), k): after 1 and 1,000 steps
  rfc7748_dh          RFC 7748 section 6.1, Alice's and Bob's keys and their shared secret
  low_order           the 7 u coordinates of X25519_LOW_ORDER_POINTS (curve25519-dalek constants.rs:91-119), whose
                      product with any scalar is zero, and their twins with bit 255 set
  pattern_0x37        x25519-dalek's byte_basepoint_matches_edwards_scalar_mul (x25519_tests.rs:5-19): the scalar
                      [0x37; 32] with byte i raised by 2 cumulatively for i = 0..31, each with x25519(k, 9); the
                      reference stores no outputs for it, so they are computed here with `cryptography`

Every vector is checked with `cryptography`'s X25519 before it is written (all outputs here are non-zero)."""
import json
import os

from cryptography.hazmat.primitives.asymmetric.x25519 import X25519PrivateKey, X25519PublicKey
from cryptography.hazmat.primitives.serialization import Encoding, PublicFormat

HERE = os.path.dirname(os.path.abspath(__file__))
BASE = bytes([9]) + bytes(31)

LADDER = [
    ("a546e36bf0527c9d3b16154b82465edd62144c0ac1fc5a18506a2244ba449ac4",
     "e6db6867583030db3594c1a424b15f7c726624ec26b3353b10a903a6d0ab1c4c",
     "c3da55379de9c6908e94ea4df28d084f32eccf03491c71f754b4075577a28552"),
    ("4b66e9d4d1b4673c5ad22691957d6af5c11b6421e0ea01d42ca4169e7918ba0d",
     "e5210f12786811d3f4b7959d0538ae2c31dbe7106fc03c3efc4cd549c715a493",
     "95cbde9476e8907d7aade45cb4b873f88b595a68799fa152e6f8f7647aac7957"),
]
ITERATED = {1: "422c8e7a6227d7bca1350b3e2bb7279f7897b87bb6854b783c60e80311ae3079",
            1000: "684cf59ba83309552800ef566f2f4d3c1c3887c49360e3875f2eb94d99532c51"}
DH = {"alice_private": "77076d0a7318a57d3c16c17251b26645df4c2f87ebc0992ab177fba51db92c2a",
      "alice_public": "8520f0098930a754748b7ddcb43ef75a0dbf3a0d26381af4eba4a98eaa9b4e6a",
      "bob_private": "5dab087e624a8a4b79e17f8b83800ee66f3bb1292618b6fd1c2f8b27ff88e0eb",
      "bob_public": "de9edb7d7b7dc1b4d35b61c2ece435373f8343c85b78674dadfc7e146f882b4f",
      "shared": "4a5d9d5ba4ce2de1728e3bf480350f25e07e21c947d19e3376f09b3c1e161742"}
LOW_ORDER = [
    "0000000000000000000000000000000000000000000000000000000000000000",
    "0100000000000000000000000000000000000000000000000000000000000000",
    "e0eb7a7c3b41b8ae1656e3faf19fc46ada098deb9c32b1fd866205165f49b800",
    "5f9c95bca3508c24b1d0b1559c83ef5b04445cc4581c8e86d8224eddd09f1157",
    "ecffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff7f",
    "edffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff7f",
    "eeffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff7f",
]


def x25519(k, u):
    return X25519PrivateKey.from_private_bytes(k).exchange(X25519PublicKey.from_public_bytes(u))


def public(k):
    return X25519PrivateKey.from_private_bytes(k).public_key().public_bytes(Encoding.Raw, PublicFormat.Raw)


def main():
    for k, u, o in LADDER:
        assert x25519(bytes.fromhex(k), bytes.fromhex(u)).hex() == o
    k = u = BASE
    for step in range(1, 1001):
        k, u = x25519(k, u), k
        if step in ITERATED:
            assert k.hex() == ITERATED[step]
    a, b = bytes.fromhex(DH["alice_private"]), bytes.fromhex(DH["bob_private"])
    assert public(a).hex() == DH["alice_public"] and public(b).hex() == DH["bob_public"]
    assert x25519(a, bytes.fromhex(DH["bob_public"])).hex() == DH["shared"]
    twins = [(bytes.fromhex(h)[:31] + bytes([bytes.fromhex(h)[31] | 0x80])).hex() for h in LOW_ORDER]
    pattern = []
    s = bytearray([0x37] * 32)
    for i in range(32):
        s[i] = (s[i] + 2) & 0xFF
        pattern.append({"scalar": bytes(s).hex(), "out": x25519(bytes(s), BASE).hex()})
    doc = {
        "rfc7748_ladder": [{"scalar": k, "u": u, "out": o} for k, u, o in LADDER],
        "rfc7748_iterated": [{"iterations": n, "out": h} for n, h in sorted(ITERATED.items())],
        "rfc7748_dh": DH,
        "low_order": LOW_ORDER,
        "low_order_bit255": twins,
        "pattern_0x37": pattern,
    }
    with open(os.path.join(HERE, "x25519.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
