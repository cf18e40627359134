"""GPU MontgomeryPoint (curve25519-dalek montgomery.rs): Scalar * MontgomeryPoint, mul_bits_be, to_edwards, the
constant-time fixed-base batch in its three output forms, and VerifyingKey::to_montgomery, through host and device
buffers, against the MontgomeryPoint oracle and against the engine's existing Edwards, Ristretto and X25519 paths, as the
reference's own tests relate them (montgomery.rs:628-701)."""
import ctypes as C
import hashlib
import random

import pytest

import montgomery_oracle as mont
import oracle_lib
import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

P = 2**255 - 19
L = pyref.L
PIECE = 1 << 16                                   # host-buffer calls of >= 2^17 items stream pieces of 2^16
N_PIECES = 2**17 + 5
BASE_U = bytes([9]) + bytes(31)
B_ENC = bytes.fromhex("5866666666666666666666666666666666666666666666666666666666666666")
RISTRETTO_B = bytes.fromhex("e2f2ae0a6abc4e71a884a961c500515f58e30b6aa582dd8db6a65945e08d2d76")
NBITS = [0, 1, 2, 254, 255, 256, 511, 512]
EDGE_SCALARS = [0, 1, L - 1, L, L + 1, 2**255 - 1]


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def mo():
    return mont.load()


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


def b32(x):
    return x.to_bytes(32, "little")


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()


def host(t, n):
    return bytes(t.cpu().numpy())[:32 * n]


def scalars(rnd, n):
    return b"".join(b32(rnd.randrange(2**255)) for _ in range(n))


def edge_us():
    us = [b32(x) for x in (0, 1, 2, 9, P - 1, P, P + 1, 2**255 - 1)]
    return us + [b32(int.from_bytes(u, "little") | 2**255) for u in us]


def to_montgomery(eng, encs):
    """EdwardsPoint::to_montgomery of CompressedEdwardsY encodings through the existing codecs"""
    rc, limbs, ok = eng.decompress_batch(b"".join(encs), len(encs))
    assert rc == 0
    return split(eng.edwards_to_montgomery_batch(limbs, len(encs)))


# ---- Scalar * MontgomeryPoint ----

@pytest.mark.parametrize("n", [1, 129, 3000])
def test_mul_parity_host_and_dev(eng, mo, n):
    rnd = random.Random(n)
    ss = scalars(rnd, n)
    us = b"".join((edge_us() + [rnd.randbytes(32) for _ in range(n)])[:n])
    want = mo.mul_bits_be_batch(ss, 32, n, 255, us, n, n)
    assert eng.montgomery_mul_batch(ss, n, us, n, n) == want
    assert host(eng.montgomery_mul_batch(dev(ss), n, dev(us), n, n, device_ptrs=True), n) == want
    # broadcast of one scalar, then of one point
    want = mo.mul_bits_be_batch(ss[:32], 32, 1, 255, us, n, n)
    assert eng.montgomery_mul_batch(ss[:32], 1, us, n, n) == want
    assert host(eng.montgomery_mul_batch(dev(ss[:32]), 1, dev(us), n, n, device_ptrs=True), n) == want
    want = mo.mul_bits_be_batch(ss, 32, n, 255, us[:32], 1, n)
    assert eng.montgomery_mul_batch(ss, n, us[:32], 1, n) == want
    assert host(eng.montgomery_mul_batch(dev(ss), n, dev(us[:32]), 1, n, device_ptrs=True), n) == want


def test_mul_across_piece_boundaries(eng, mo):
    n = N_PIECES
    rnd = random.Random(11)
    ss, us = scalars(rnd, n), rnd.randbytes(32 * n)
    want = mo.mul_bits_be_batch(ss, 32, n, 255, us, n, n)
    assert eng.montgomery_mul_batch(ss, n, us, n, n) == want
    assert host(eng.montgomery_mul_batch(dev(ss), n, dev(us), n, n, device_ptrs=True), n) == want
    assert eng.last_call_ms() > 0


def test_mul_edge_scalars(eng, mo):
    us = edge_us() + [BASE_U]
    for s in EDGE_SCALARS:
        n = len(us)
        want = mo.mul_bits_be_batch(b32(s), 32, 1, 255, b"".join(us), n, n)
        assert eng.montgomery_mul_batch(b32(s), 1, b"".join(us), n, n) == want


# ---- mul_bits_be ----

@pytest.mark.parametrize("nbits", NBITS)
def test_mul_bits_be_parity(eng, mo, nbits):
    rnd = random.Random(100 + nbits)
    n = 700
    us = b"".join(edge_us() + [rnd.randbytes(32) for _ in range(n - len(edge_us()))])
    for int_bytes in sorted({1, 31, 33, 64, max(1, (nbits + 7) // 8)}):
        if nbits > 8 * int_bytes:
            continue
        ints = rnd.randbytes(int_bytes * n)
        want = mo.mul_bits_be_batch(ints, int_bytes, n, nbits, us, n, n)
        assert eng.montgomery_mul_bits_be_batch(ints, int_bytes, n, nbits, us, n, n) == want, int_bytes
        want = mo.mul_bits_be_batch(ints[:int_bytes], int_bytes, 1, nbits, us, n, n)
        assert eng.montgomery_mul_bits_be_batch(ints[:int_bytes], int_bytes, 1, nbits, us, n, n) == want
        want = mo.mul_bits_be_batch(ints, int_bytes, n, nbits, us[:32], 1, n)
        assert eng.montgomery_mul_bits_be_batch(ints, int_bytes, n, nbits, us[:32], 1, n) == want
    if nbits == 0:
        assert eng.montgomery_mul_bits_be_batch(b"\xff", 1, 1, 0, us, n, n) == bytes(32 * n)


def test_mul_bits_be_across_piece_boundaries(eng, mo):
    n, int_bytes, nbits = N_PIECES, 33, 263                      # an odd integer size: unaligned items
    rnd = random.Random(12)
    ints, us = rnd.randbytes(int_bytes * n), rnd.randbytes(32 * n)
    want = mo.mul_bits_be_batch(ints, int_bytes, n, nbits, us, n, n)
    assert eng.montgomery_mul_bits_be_batch(ints, int_bytes, n, nbits, us, n, n) == want


def test_scalar_times_to_montgomery_is_to_montgomery_of_product(eng, orc):
    """montgomery.rs:628-645: s * to_montgomery(P) == to_montgomery(s * P)"""
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(13)
    n = 200
    pts = [orc.compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())) for _ in range(n)]
    ss = [b32(rnd.randrange(2**255)) for _ in range(n)]
    prods = pkg.EdwardsPoint.mul_batch(ss, pts, engine=eng)
    got = split(eng.montgomery_mul_batch(b"".join(ss), n, b"".join(to_montgomery(eng, pts)), n, n))
    assert got == to_montgomery(eng, prods)


def test_mul_bits_be_512_is_wide_scalar_product(eng, orc):
    """montgomery.rs:650-672: mul_bits_be(b, u(P)) == to_montgomery(from_bytes_mod_order_wide(b) P) for 512-bit b"""
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(14)
    n = 200
    pts = [orc.compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())) for _ in range(n)]
    wide = rnd.randbytes(64 * n)
    red = split(eng.scalar_from_wide_batch(wide, n))
    want = to_montgomery(eng, pkg.EdwardsPoint.mul_batch(red, pts, engine=eng))
    assert split(eng.montgomery_mul_bits_be_batch(wide, 64, n, 512, b"".join(to_montgomery(eng, pts)), n, n)) == want


def test_mul_bits_be_commutes_on_curve_and_twist(eng):
    """montgomery.rs:676-701: b1 (b2 P) == b2 (b1 P) for random u, twist points included"""
    rnd = random.Random(15)
    n = 1000
    us, b1, b2 = rnd.randbytes(32 * n), rnd.randbytes(64 * n), rnd.randbytes(64 * n)
    p1 = eng.montgomery_mul_bits_be_batch(b1, 64, n, 512, us, n, n)
    p2 = eng.montgomery_mul_bits_be_batch(b2, 64, n, 512, us, n, n)
    assert eng.montgomery_mul_bits_be_batch(b2, 64, n, 512, p1, n, n) == eng.montgomery_mul_bits_be_batch(b1, 64, n, 512, p2, n, n)


# ---- to_edwards ----

def test_to_edwards_parity(eng, mo, orc):
    rnd = random.Random(16)
    pts = [orc.compress(orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint())) for _ in range(500)]
    us = to_montgomery(eng, pts) + [rnd.randbytes(32) for _ in range(500)] + edge_us()
    signs = bytes(rnd.randrange(256) for _ in us)
    n = len(us)
    want, ok = mo.to_edwards_batch(b"".join(us), signs, n)
    rc, got, gok = eng.montgomery_to_edwards_batch(b"".join(us), signs, n)
    assert got == want and gok == ok and rc == 1 and 0 < sum(ok) < n
    rc, got, gok = eng.montgomery_to_edwards_batch(b"".join(us[:500]), signs[:500], 500)
    assert rc == 0 and gok == b"\x01" * 500


def test_to_edwards_across_piece_boundaries(eng, mo):
    n = N_PIECES
    rnd = random.Random(17)
    us, signs = rnd.randbytes(32 * n), rnd.randbytes(n)
    want, ok = mo.to_edwards_batch(us, signs, n)
    rc, got, gok = eng.montgomery_to_edwards_batch(us, signs, n)
    assert got == want and gok == ok and rc == 1


def test_to_edwards_reference_cases(eng):
    import curve25519_dalek_b200 as pkg
    MP = pkg.MontgomeryPoint
    minus_B = pyref.compress(pyref.neg(pyref.B))
    assert MP.to_edwards_batch([BASE_U] * 4, [0, 1, 2, 255], engine=eng) == [B_ENC, minus_B, B_ENC, minus_B]
    minus_one = [b32(P - 1), b32((P - 1) | 2**255)]
    assert MP.to_edwards_batch(minus_one + [b32(2)], 0, engine=eng) == [None, None, None]
    assert MP.to_edwards_batch(minus_one, 1, engine=eng) == [None, None]
    assert MP.to_edwards_batch([b32(18), b"\xff" * 32], 1, engine=eng) == MP.to_edwards_batch([b32(18)] * 2, 1, engine=eng)
    assert MP.to_edwards_batch([bytes(32)] * 2, [0, 1], engine=eng) == [b32(P - 1)] * 2     # (0, -1) with either sign


def test_to_edwards_round_trips_random_and_torsion_points(eng, orc):
    rnd = random.Random(18)
    tors = torsion_points(orc)
    pts = [orc.scalarmul(b32(rnd.randrange(L)), orc.basepoint()) for _ in range(100)]
    pts += tors + [orc.add(p, tors[i % 7]) for i, p in enumerate(pts[:50])]
    encs = [orc.compress(p) for p in pts]
    us = to_montgomery(eng, encs)
    signs = bytes(e[31] >> 7 for e in encs)
    rc, got, ok = eng.montgomery_to_edwards_batch(b"".join(us), signs, len(encs))
    assert rc == 0 and split(got) == encs


# ---- constant-time fixed base ----

def _mul_base_cases(rnd, n):
    return b"".join([b32(s) for s in EDGE_SCALARS] + [b32(rnd.randrange(2**255)) for _ in range(n - len(EDGE_SCALARS))])


@pytest.mark.parametrize("n", [1000, 16384 + 3])
def test_mul_base_matches_mul_batch_of_b(eng, mo, n):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(n)
    ss = _mul_base_cases(rnd, n)
    ed = eng.mul_base_ct_batch(ss, n, pkg.POINTS_COMPRESSED)
    assert ed == eng.mul_batch(ss, n, B_ENC, 1, n)[1]
    assert ed == eng.mul_base_batch(ss, n)[1]                                    # the variable-time table
    ri = eng.mul_base_ct_batch(ss, n, pkg.POINTS_RISTRETTO)
    assert ri == eng.mul_batch(ss, n, RISTRETTO_B, 1, n, point_fmt=pkg.POINTS_RISTRETTO)[1]
    mu = eng.mul_base_ct_batch(ss, n, pkg.POINTS_MONTGOMERY)
    assert mu == eng.montgomery_mul_batch(ss, n, BASE_U, 1, n)
    assert mu == b"".join(to_montgomery(eng, split(ed)))
    k = rnd.randbytes(32 * n)
    ec = eng.mul_base_ct_batch(k, n, pkg.POINTS_COMPRESSED, clamped=True)
    assert ec == eng.mul_batch(k, n, B_ENC, 1, n, clamped=True)[1]
    mc = eng.mul_base_ct_batch(k, n, pkg.POINTS_MONTGOMERY, clamped=True)
    assert mc == eng.x25519_public_keys(k, n)
    idx = list(range(len(EDGE_SCALARS))) + [n - 1]
    sub = b"".join(ss[32 * i:32 * i + 32] for i in idx)
    for fmt, got in ((mont.FMT_COMPRESSED, ed), (mont.FMT_RISTRETTO, ri), (mont.FMT_MONTGOMERY, mu)):
        assert b"".join(got[32 * i:32 * i + 32] for i in idx) == mo.mul_base_batch(sub, len(idx), fmt)


def test_mul_base_across_piece_boundaries(eng, mo):
    import curve25519_dalek_b200 as pkg
    n = N_PIECES
    rnd = random.Random(19)
    ss = scalars(rnd, n)
    for fmt in (pkg.POINTS_COMPRESSED, pkg.POINTS_RISTRETTO, pkg.POINTS_MONTGOMERY):
        assert eng.mul_base_ct_batch(ss, n, fmt) == mo.mul_base_batch(ss, n, fmt), fmt


def test_mul_base_python_wrappers(eng, mo):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(20)
    ss = [b32(s) for s in EDGE_SCALARS] + [b32(rnd.randrange(2**255)) for _ in range(10)]
    assert pkg.EdwardsPoint.mul_base_batch(ss, engine=eng) == [mo.mul_base(s, mont.FMT_COMPRESSED) for s in ss]
    assert pkg.RistrettoPoint.mul_base_batch(ss, engine=eng) == [mo.mul_base(s, mont.FMT_RISTRETTO) for s in ss]
    assert pkg.MontgomeryPoint.mul_base_batch(ss, engine=eng) == [mo.mul_base(s, mont.FMT_MONTGOMERY) for s in ss]
    assert pkg.EdwardsPoint.mul_base_batch(ss[2], engine=eng) == mo.mul_base(ss[2], mont.FMT_COMPRESSED)
    ks = [rnd.randbytes(32) for _ in range(10)] + [b"\xff" * 32]
    assert pkg.EdwardsPoint.mul_base_clamped_batch(ks, engine=eng) == [mo.mul_base(k, mont.FMT_COMPRESSED, True) for k in ks]
    assert pkg.MontgomeryPoint.mul_base_clamped_batch(ks, engine=eng) == pkg.x25519_public_keys(ks, engine=eng)
    # montgomery.rs:704-711: mul_base_clamped == X25519_BASEPOINT.mul_clamped, on [0xff; 32] and random bytes
    assert pkg.MontgomeryPoint.mul_base_clamped_batch(ks, engine=eng) == pkg.MontgomeryPoint.mul_clamped_batch(ks, BASE_U, engine=eng)
    for bad in (b32(2**255), b"\xff" * 32):
        for fn in (pkg.EdwardsPoint.mul_base_batch, pkg.RistrettoPoint.mul_base_batch, pkg.MontgomeryPoint.mul_base_batch):
            with pytest.raises(ValueError):
                fn([bad], engine=eng)


def test_montgomery_python_wrappers(eng, mo):
    import curve25519_dalek_b200 as pkg
    MP = pkg.MontgomeryPoint
    rnd = random.Random(21)
    ss = [b32(rnd.randrange(2**255)) for _ in range(5)]
    us = [rnd.randbytes(32) for _ in range(5)]
    assert MP.mul_batch(ss, us, engine=eng) == [mo.mul(s, u) for s, u in zip(ss, us)]
    assert MP.mul_batch(ss[0], us[0], engine=eng) == mo.mul(ss[0], us[0])
    assert MP.mul_batch(ss[0], us, engine=eng) == [mo.mul(ss[0], u) for u in us]
    ints = [rnd.randbytes(40) for _ in range(5)]
    assert MP.mul_bits_be_batch(ints, 300, us, engine=eng) == [mo.mul_bits_be(u, b, 300) for b, u in zip(ints, us)]
    assert MP.mul_bits_be_batch(ints, 300, us[0], engine=eng) == [mo.mul_bits_be(us[0], b, 300) for b in ints]
    ks = [rnd.randbytes(32) for _ in range(5)]
    assert MP.mul_clamped_batch(ks, us, engine=eng) == pkg.x25519(ks, us, engine=eng)
    assert MP.mul_clamped_batch(ks[0], us, engine=eng) == pkg.x25519([ks[0]] * 5, us, engine=eng)
    with pytest.raises(ValueError):
        MP.mul_batch([b32(2**255)], us[:1], engine=eng)
    with pytest.raises(ValueError):
        MP.mul_bits_be_batch(ints, 321, us, engine=eng)
    with pytest.raises(ValueError):
        MP.mul_bits_be_batch([bytes(65)], 8, us[:1], engine=eng)
    with pytest.raises(ValueError):
        MP.mul_batch(ss[:2], us[:3], engine=eng)


# ---- VerifyingKey::to_montgomery ----

def test_ed25519_to_montgomery(eng):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(22)
    seeds = [rnd.randbytes(32) for _ in range(300)]
    vks = pkg.ed25519_verifying_keys(seeds, engine=eng)
    want = pkg.x25519_public_keys([hashlib.sha512(s).digest()[:32] for s in seeds], engine=eng)
    assert pkg.ed25519_to_montgomery(vks, engine=eng) == want
    bad = next(b32(y) for y in range(2, 100) if pyref.decompress(b32(y)) is None)
    assert pkg.ed25519_to_montgomery([vks[0], bad, vks[1]], engine=eng) == [want[0], None, want[1]]
    assert pkg.ed25519_to_montgomery(vks[2], engine=eng) == want[2]


# ---- argument rules ----

def test_invalid_arguments(eng):
    import curve25519_dalek_b200 as pkg
    lib, h = eng.lib, eng.h
    E = -1
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    out = (C.c_uint8 * 4096)()
    o = C.addressof(out)
    # Scalar * MontgomeryPoint
    assert lib.dalek_b200_montgomery_mul_batch(h, p, 2, p, 5, 5, o) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, p, 5, p, 3, 5, o) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, None, 1, p, 1, 1, o) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, p, 1, None, 1, 1, o) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, p, 1, p, 1, 1, None) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, None, 0, None, 0, 0, None) == 0
    top = (C.c_uint8 * 64)(*([0] * 31 + [0x80] + [0] * 32))
    assert lib.dalek_b200_montgomery_mul_batch(h, C.addressof(top), 1, p, 1, 1, o) == E
    assert lib.dalek_b200_montgomery_mul_batch(h, p, 2, p, 2, 2, o) == 0
    with pytest.raises(pkg.EngineError):
        eng.montgomery_mul_batch(dev(bytes(top)), 2, dev(bytes(64)), 2, 2, device_ptrs=True)
    assert lib.dalek_b200_montgomery_mul_batch_dev(h, None, 1, p, 1, 1, o) == E
    assert lib.dalek_b200_montgomery_mul_batch_dev(h, p, 2, p, 1, 3, o) == E
    assert lib.dalek_b200_montgomery_mul_batch_dev(h, None, 0, None, 0, 0, None) == 0
    # mul_bits_be
    fn = lib.dalek_b200_montgomery_mul_bits_be_batch
    assert fn(h, p, 0, 1, 0, p, 1, 1, o) == E
    assert fn(h, p, 65, 1, 8, p, 1, 1, o) == E
    assert fn(h, p, 4, 1, 33, p, 1, 1, o) == E
    assert fn(h, p, 4, 2, 32, p, 1, 3, o) == E
    assert fn(h, p, 4, 1, 32, p, 2, 3, o) == E
    assert fn(h, None, 4, 1, 32, p, 1, 1, o) == E
    assert fn(h, p, 4, 1, 32, p, 1, 1, None) == E
    assert fn(h, p, 4, 1, 32, p, 1, 1, o) == 0
    assert fn(h, p, 64, 1, 512, p, 1, 1, o) == 0
    assert fn(h, None, 4, 0, 32, None, 0, 0, None) == 0
    # to_edwards
    assert lib.dalek_b200_montgomery_to_edwards_batch(h, None, p, 1, o, None) == E
    assert lib.dalek_b200_montgomery_to_edwards_batch(h, p, None, 1, o, None) == E
    assert lib.dalek_b200_montgomery_to_edwards_batch(h, p, p, 1, None, None) == E
    assert lib.dalek_b200_montgomery_to_edwards_batch(h, None, None, 0, None, None) == 0
    # constant-time fixed base
    fn = lib.dalek_b200_mul_base_ct_batch
    assert fn(h, p, 1, pkg.POINTS_EXTENDED, 0, o) == E
    assert fn(h, p, 1, 4, 0, o) == E
    assert fn(h, p, 1, pkg.POINTS_RISTRETTO, 1, o) == E
    assert fn(h, p, 1, pkg.POINTS_COMPRESSED, 2, o) == E
    assert fn(h, None, 1, pkg.POINTS_COMPRESSED, 0, o) == E
    assert fn(h, p, 1, pkg.POINTS_COMPRESSED, 0, None) == E
    assert fn(h, C.addressof(top), 1, pkg.POINTS_MONTGOMERY, 0, o) == E
    assert fn(h, C.addressof(top), 1, pkg.POINTS_MONTGOMERY, 1, o) == 0              # clamped: any 32 bytes
    assert fn(h, None, 0, pkg.POINTS_COMPRESSED, 0, None) == 0
    # the context stays usable
    assert eng.montgomery_mul_batch(b32(1), 1, BASE_U, 1, 1) == BASE_U
