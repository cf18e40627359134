"""GPU X25519: x25519(k, u) (x25519-dalek x25519.rs:390-392) through host and device buffers, PublicKey::from
(x25519.rs:105-110) through the fixed-base comb, and EdwardsPoint::to_montgomery_batch (C/edwards.rs:592-612), against
the golden vectors, the X25519 oracle, `cryptography` and the engine's own Edwards paths."""
import ctypes as C
import json
import os
import random

import pytest

import pyref
import x25519_oracle
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = bytes([9]) + bytes(31)
PIECE = 1 << 16                                   # host-buffer calls of >= 2^17 items stream pieces of 2^16


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def xo():
    return x25519_oracle.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "x25519.json")) as f:
        return json.load(f)


def b32(x):
    return x.to_bytes(32, "little")


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()


def x_dev(eng, ks, us, n):
    out, flags = eng.x25519_batch(dev(ks), dev(us), n, device_ptrs=True, want_contributory=True)
    return bytes(out.cpu().numpy())[:32 * n], bytes(flags.cpu().numpy())[:n]


def test_golden_vectors_host_and_dev(eng, golden):
    cases = [(v["scalar"], v["u"], v["out"]) for v in golden["rfc7748_ladder"]]
    dh = golden["rfc7748_dh"]
    cases += [(dh["alice_private"], BASE.hex(), dh["alice_public"]), (dh["bob_private"], BASE.hex(), dh["bob_public"]),
              (dh["alice_private"], dh["bob_public"], dh["shared"]), (dh["bob_private"], dh["alice_public"], dh["shared"])]
    cases += [(v["scalar"], BASE.hex(), v["out"]) for v in golden["pattern_0x37"]]
    ks = b"".join(bytes.fromhex(c[0]) for c in cases)
    us = b"".join(bytes.fromhex(c[1]) for c in cases)
    want = [bytes.fromhex(c[2]) for c in cases]
    out, flags = eng.x25519_batch(ks, us, len(cases), want_contributory=True)
    assert split(out) == want and flags == bytes([1]) * len(cases)
    out, flags = x_dev(eng, ks, us, len(cases))
    assert split(out) == want and flags == bytes([1]) * len(cases)
    pks = split(eng.x25519_public_keys(b"".join(bytes.fromhex(c[0]) for c in cases[2:4] + cases[6:]), len(cases) - 4))
    assert pks == want[2:4] + want[6:]


def test_iterated_vector_one_call_per_step(eng, golden):
    want = {v["iterations"]: v["out"] for v in golden["rfc7748_iterated"]}
    k = u = BASE
    for step in range(1, max(want) + 1):
        out, _ = eng.x25519_batch(k, u, 1)
        k, u = out, k
        if step in want:
            assert k.hex() == want[step]
    k = u = dev(BASE)
    for step in range(1, max(want) + 1):
        out, _ = eng.x25519_batch(k, u, 1, device_ptrs=True)
        k, u = out[:32], k
        if step in want:
            assert bytes(k.cpu().numpy()).hex() == want[step]


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 2**16 - 1, 2**16 + 1, 2**17 + 3])
def test_random_batches_match_oracle(eng, xo, n):
    rnd = random.Random(n)
    ks, us = rnd.randbytes(32 * n), rnd.randbytes(32 * n)
    out, flags = eng.x25519_batch(ks, us, n, want_contributory=True)
    dout, dflags = x_dev(eng, ks, us, n) if n else (b"", b"")
    assert len(out) == 32 * n and dout == out and dflags == flags
    idx = range(n) if n <= 2**14 else sorted(set(rnd.randrange(n) for _ in range(4096)) | {i for i in (0, PIECE - 1, PIECE, n - 1) if i < n})
    ok = xo.x25519_batch(b"".join(ks[32 * i:32 * i + 32] for i in idx), b"".join(us[32 * i:32 * i + 32] for i in idx))
    for j, i in enumerate(idx):
        assert out[32 * i:32 * i + 32] == ok[32 * j:32 * j + 32], i
        assert flags[i] == (ok[32 * j:32 * j + 32] != bytes(32))
    if n:
        ms, launches = eng.last_kernel_ms()
        assert ms > 0 and launches == 1 and eng.last_call_ms() > 0


def test_diffie_hellman_commutes_over_a_large_batch(eng):
    n = 2**17
    rnd = random.Random(7)
    a, b = rnd.randbytes(32 * n), rnd.randbytes(32 * n)
    A, _ = eng.x25519_batch(a, BASE * n, n)
    B, _ = eng.x25519_batch(b, BASE * n, n)
    s1, _ = eng.x25519_batch(a, B, n)
    s2, _ = eng.x25519_batch(b, A, n)
    assert s1 == s2 and len(set(split(s1[:32 * 1024]))) == 1024


def test_low_order_points_at_piece_boundaries(eng, golden):
    n = 2**17 + 3
    rnd = random.Random(8)
    ks = rnd.randbytes(32 * n)
    us = bytearray(rnd.randbytes(32 * n))
    for i in range(n):                            # random u on the curve or its twin: never a low-order point
        us[32 * i] |= 0x40
    low = [bytes.fromhex(h) for h in golden["low_order"] + golden["low_order_bit255"]]
    where = [0, 1, 127, 128, 777, 99999, PIECE - 1, PIECE, PIECE + 1, 2 * PIECE - 1, 2 * PIECE, 2 * PIECE + 1, n - 1]
    for j, i in enumerate(where):
        us[32 * i:32 * i + 32] = low[j % len(low)]
    us = bytes(us)
    for out, flags in (eng.x25519_batch(ks, us, n, want_contributory=True), x_dev(eng, ks, us, n)):
        zero = {i for i in range(n) if out[32 * i:32 * i + 32] == bytes(32)}
        assert zero == set(where)
        assert [i for i in range(n) if flags[i] == 0] == sorted(where)


def test_public_keys(eng, xo, oracle, golden):
    x = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.x25519")
    from cryptography.hazmat.primitives.serialization import Encoding, PublicFormat
    n = 2**17 + 3
    rnd = random.Random(9)
    ks = bytearray(rnd.randbytes(32 * n))
    ks[:64] = bytes(32) + b"\xff" * 32
    ks = bytes(ks)
    pks = eng.x25519_public_keys(ks, n)
    ladder, _ = eng.x25519_batch(ks, BASE * n, n)
    assert pks == ladder
    assert eng.last_call_ms() > 0
    idx = sorted(set(rnd.randrange(n) for _ in range(4096)) | {0, 1, PIECE - 1, PIECE, n - 1})
    for i in idx[:512]:
        k = ks[32 * i:32 * i + 32]
        assert pks[32 * i:32 * i + 32] == xo.public_key(k)
        pk = x.X25519PrivateKey.from_private_bytes(k).public_key().public_bytes(Encoding.Raw, PublicFormat.Raw)
        assert pks[32 * i:32 * i + 32] == pk
    dh = golden["rfc7748_dh"]
    got = eng.x25519_public_keys(bytes.fromhex(dh["alice_private"] + dh["bob_private"]), 2)
    assert got.hex() == dh["alice_public"] + dh["bob_public"]
    # the two existing Edwards paths chained: EdwardsPoint::mul_base then to_montgomery_batch
    m = 3000
    clamped = b"".join(xo.clamp(ks[32 * i:32 * i + 32]) for i in range(m))
    limbs, _ = eng.mul_base_batch(clamped, m, want_compressed=False)
    assert eng.edwards_to_montgomery_batch(limbs, m) == pks[:32 * m]


def test_to_montgomery_batch(eng, xo, oracle):
    rnd = random.Random(10)
    B = oracle.basepoint()
    pts = [oracle.identity()] + torsion_points(oracle)
    pts += [oracle.add(oracle.scalarmul(b32(rnd.randrange(1, pyref.L)), B), pts[rnd.randrange(8)]) for _ in range(60)]
    pts += [oracle.identity()] * 3 + torsion_points(oracle)
    n = len(pts)
    ext = (C.c_uint64 * (20 * n))()
    for i, p in enumerate(pts):
        lam = 1 if i == 0 else rnd.randrange(2, pyref.p)       # Z != 1 for every point but the first
        xyzt = [sum(v << (51 * k) for k, v in enumerate(oracle.p3_limbs(p)[5 * c:5 * c + 5])) * lam % pyref.p for c in range(4)]
        for c in range(4):
            for k in range(5):
                ext[20 * i + 5 * c + k] = (xyzt[c] >> (51 * k)) & (2**51 - 1)
    got = split(eng.edwards_to_montgomery_batch(ext, n))
    assert got == [xo.to_montgomery(list(ext[20 * i:20 * i + 20])) for i in range(n)]
    assert got[0] == bytes(32) and got[n - 8] == bytes(32)            # the identity
    assert got[4] == bytes(32)                                        # 4T8 = (0, -1), order 2
    assert got[2] == b32(1) and got[6] == b32(1)                      # 2T8, 6T8 = (+-sqrt(-1), 0), order 4


def test_zero_and_invalid_arguments(eng):
    lib, h = eng.lib, eng.h
    for fn, args in ((lib.dalek_b200_x25519_batch, (None, None, 0, None, None)),
                     (lib.dalek_b200_x25519_batch_dev, (None, None, 0, None, None)),
                     (lib.dalek_b200_x25519_public_keys, (None, 0, None)),
                     (lib.dalek_b200_edwards_to_montgomery_batch, (None, 0, None))):
        assert fn(h, *args) == 0
    buf = (C.c_uint8 * 64)()
    a = C.addressof(buf)
    assert lib.dalek_b200_x25519_batch(h, a, None, 1, a, None) == -1
    assert lib.dalek_b200_x25519_batch(h, a, a, 1, None, None) == -1
    assert lib.dalek_b200_x25519_batch_dev(h, None, a, 1, a, None) == -1
    assert lib.dalek_b200_x25519_public_keys(h, a, 1, None) == -1
    assert lib.dalek_b200_edwards_to_montgomery_batch(h, None, 1, a) == -1


def test_module_level_functions(eng, xo, oracle, golden):
    import curve25519_dalek_b200 as pkg
    dh = {k: bytes.fromhex(v) for k, v in golden["rfc7748_dh"].items()}
    assert pkg.X25519_BASEPOINT_BYTES == BASE
    assert pkg.x25519(dh["alice_private"], dh["bob_public"], engine=eng) == dh["shared"]
    assert pkg.x25519([dh["alice_private"], dh["bob_private"]], [BASE, BASE], engine=eng) == [dh["alice_public"], dh["bob_public"]]
    assert pkg.x25519_public_keys([dh["alice_private"], dh["bob_private"]], engine=eng) == [dh["alice_public"], dh["bob_public"]]
    assert pkg.x25519_public_keys(dh["bob_private"], engine=eng) == dh["bob_public"]
    limbs, _ = eng.mul_base_batch(xo.clamp(dh["alice_private"]) + xo.clamp(dh["bob_private"]), 2, want_compressed=False)
    assert pkg.EdwardsPoint.to_montgomery_batch(limbs, engine=eng) == [dh["alice_public"], dh["bob_public"]]
