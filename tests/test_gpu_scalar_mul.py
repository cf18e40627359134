"""GPU variable-base scalar multiplication: dalek_b200_mul_batch / _dev (EdwardsPoint * Scalar, mul_clamped,
RistrettoPoint * Scalar, BasepointTable::create(P) * s) and dalek_b200_edwards_torsion_batch (is_small_order,
is_torsion_free), against the golden vectors of tests/golden/scalar_mul.json and the C oracle."""
import json
import os
import random

import pytest

import oracle_lib
import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
DALEK_NONE, INVALID = 1, -1
COMB_MIN = 16384                                  # varmul.cu VARMUL_COMB_MIN
PIECE = 1 << 16


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def orc():
    return oracle_lib.load()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json")) as f:
        return json.load(f)


def b32(x):
    return x.to_bytes(32, "little")


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()


def clamp(b):
    b = bytearray(b)
    b[0] &= 248
    b[31] &= 127
    b[31] |= 64
    return bytes(b)


def run(eng, ss, ps, n, fmt=COMPRESSED, clamped=False, device=False):
    """(rc, outputs, ok) through host or device buffers"""
    if device:
        rc, out, ok = eng.mul_batch(dev(b"".join(ss)), len(ss), dev(b"".join(ps)), len(ps), n, fmt, clamped=clamped,
                                    device_ptrs=True, want_ok=True)
        return rc, split(bytes(out.cpu().numpy())[:32 * n]), bytes(ok.cpu().numpy())[:n]
    rc, out, ok = eng.mul_batch(b"".join(ss), len(ss), b"".join(ps), len(ps), n, fmt, clamped=clamped, want_ok=True)
    return rc, split(out), ok


def encode(orc, P, fmt):
    return orc.ristretto_compress(P) if fmt == RISTRETTO else orc.compress(P)


def point_input(orc, P, fmt):
    if fmt == EXTENDED:
        return b"".join(int(v).to_bytes(8, "little") for v in orc.p3_limbs(P))
    return encode(orc, P, fmt)


def want(orc, s, P, fmt, clamped=False):
    return encode(orc, orc.scalarmul(clamp(s) if clamped else s, P), fmt)


def random_points(orc, rnd, k):
    B = orc.basepoint()
    return [orc.scalarmul(b32(rnd.randrange(1, L)), B) for _ in range(k)]


@pytest.mark.parametrize("device", [False, True])
def test_golden_vectors(eng, golden, device):
    a, base = bytes.fromhex(golden["A_SCALAR"]), bytes.fromhex(golden["BASEPOINT"])
    aB = bytes.fromhex(golden["A_TIMES_BASEPOINT"])
    order = bytes.fromhex(golden["BASEPOINT_ORDER"])
    rc, out, ok = run(eng, [a, a, order], [base, aB, base], 3, device=device)
    assert rc == 0 and ok == b"\x01" * 3
    assert [o.hex() for o in out] == [golden["A_TIMES_BASEPOINT"], golden["A_TIMES_A_TIMES_BASEPOINT"], golden["IDENTITY"]]
    torsion = [bytes.fromhex(t["compressed"]) for t in golden["EIGHT_TORSION"]]
    rc, out, _ = run(eng, [b32(8)], torsion, 8, device=device)
    assert rc == 0 and [o.hex() for o in out] == [golden["IDENTITY"]] * 8


@pytest.mark.parametrize("fmt", [COMPRESSED, EXTENDED, RISTRETTO])
@pytest.mark.parametrize("n", [1, 7, 1000])
@pytest.mark.parametrize("shape", ["each", "one_scalar", "one_point", "one_each"])
def test_formats_and_shapes(eng, orc, fmt, n, shape):
    rnd = random.Random(n * 10 + fmt)
    ns = 1 if shape in ("one_scalar", "one_each") else n
    npts = 1 if shape in ("one_point", "one_each") else n
    pts = random_points(orc, rnd, npts)
    ss = [b32(rnd.randrange(L)) for _ in range(ns)]
    for device in (False, True):
        rc, out, ok = run(eng, ss, [point_input(orc, P, fmt) for P in pts], n, fmt, device=device)
        assert rc == 0 and ok == b"\x01" * n
        for i in range(n):
            assert out[i] == want(orc, ss[i % ns], pts[i % npts], fmt), (i, device)


def test_piece_boundary(eng, orc):
    n = 2 * PIECE + 3
    rnd = random.Random(5)
    pool = random_points(orc, rnd, 64)
    pts = [pool[rnd.randrange(64)] for _ in range(n)]
    ss = [b32(rnd.randrange(L)) for _ in range(n)]
    rc, out, ok = run(eng, ss, [orc.compress(P) for P in pts], n)
    assert rc == 0 and ok == b"\x01" * n
    idx = set(range(200)) | set(range(n - 200, n)) | set(range(PIECE - 100, PIECE + 100)) | set(range(2 * PIECE - 100, 2 * PIECE + 3))
    idx |= {rnd.randrange(n) for _ in range(1000)}
    for i in sorted(idx):
        assert out[i] == want(orc, ss[i], pts[i], COMPRESSED), i


@pytest.mark.parametrize("fmt", [COMPRESSED, EXTENDED, RISTRETTO])
def test_shared_point_path_at_cutoff(eng, orc, fmt):
    rnd = random.Random(6 + fmt)
    P = random_points(orc, rnd, 1)[0]
    ss = [b32(rnd.randrange(L)) for _ in range(COMB_MIN)]
    pin = point_input(orc, P, fmt)
    rc0, below, _ = run(eng, ss[:COMB_MIN - 1], [pin], COMB_MIN - 1, fmt)   # per-item path
    rc1, at, ok = run(eng, ss, [pin], COMB_MIN, fmt)                          # comb path
    rc2, each, _ = run(eng, ss, [pin] * COMB_MIN, COMB_MIN, fmt)              # per-item path, the point repeated
    assert rc0 == rc1 == rc2 == 0 and ok == b"\x01" * COMB_MIN
    assert at[:COMB_MIN - 1] == below and at == each
    for i in list(range(20)) + [rnd.randrange(COMB_MIN) for _ in range(50)] + [COMB_MIN - 1]:
        assert at[i] == want(orc, ss[i], P, fmt)
    rc, at_dev, _ = run(eng, ss, [pin], COMB_MIN, fmt, device=True)
    assert rc == 0 and at_dev == at


@pytest.mark.parametrize("n", [7, COMB_MIN])
def test_clamped_scalars(eng, orc, n):
    rnd = random.Random(7)
    P = random_points(orc, rnd, 1)[0]
    ss = [b"\xff" * 32, bytes(32), b"\x80" * 32] + [rnd.randbytes(32) for _ in range(n - 3)]
    for pts in ([orc.compress(P)], [orc.compress(P)] * n):
        for device in (False, True):
            rc, out, _ = run(eng, ss, pts, n, clamped=True, device=device)
            assert rc == 0
            for i in sorted(set(range(min(n, 10))) | {n - 1}):
                assert out[i] == want(orc, ss[i], P, COMPRESSED, clamped=True)


def test_ristretto_coset_invariance(eng, orc):
    rnd = random.Random(8)
    tors = torsion_points(orc)
    four = [orc.identity(), tors[1], tors[3], tors[5]]          # the 4-torsion: orders 1, 4, 2, 4
    Ps = random_points(orc, rnd, 5)
    ss = [b32(rnd.randrange(L)) for _ in range(5)]
    for P, s in zip(Ps, ss):
        encs = [orc.ristretto_compress(orc.add(P, T)) for T in four]
        assert len(set(encs)) == 1
        rc, out, _ = run(eng, [s], encs, 4, RISTRETTO)
        assert rc == 0 and len(set(out)) == 1 and out[0] == want(orc, s, P, RISTRETTO)
        # the extended coordinates of P + T for each 4-torsion T are different representatives of one Ristretto point
        rc, out_e, _ = run(eng, [s], [point_input(orc, orc.add(P, T), EXTENDED) for T in four], 4, EXTENDED)
        assert rc == 0
        assert [orc.ristretto_compress(orc.decompress(o)) for o in out_e] == [out[0]] * 4


def test_ristretto_rejection_classes(eng, orc):
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        classes = json.load(f)["classes"]
    for cls in ("noncanonical", "negative", "nonsquare", "t_negative", "y_zero", "valid"):
        encs = [bytes.fromhex(v["s"]) for v in classes[cls]]
        n = len(encs)
        for device in (False, True):
            rc, out, ok = run(eng, [b32(5)], encs, n, RISTRETTO, device=device)
            if cls == "valid":
                assert rc == 0 and ok == b"\x01" * n
                assert out == [want(orc, b32(5), orc.ristretto_decompress(e), RISTRETTO) for e in encs]
            else:
                assert rc == DALEK_NONE and ok == bytes(n) and out == [bytes(32)] * n, cls


def test_undecodable_points(eng, orc):
    rnd = random.Random(9)
    pts = random_points(orc, rnd, 6)
    encs = [orc.compress(P) for P in pts]
    encs[2] = b32(2)                                             # y = 2 is not on the curve
    encs[4] = b32(2)
    ss = [b32(rnd.randrange(L)) for _ in range(6)]
    for device in (False, True):
        rc, out, ok = run(eng, ss, encs, 6, device=device)
        assert rc == DALEK_NONE and ok == bytes([1, 1, 0, 1, 0, 1])
        for i in range(6):
            assert out[i] == (b32(1) if i in (2, 4) else want(orc, ss[i], pts[i], COMPRESSED))
    # one undecodable point for a whole batch, on both sides of the comb cutoff
    for n in (5, COMB_MIN):
        rc, out, ok = run(eng, [b32(3)], [b32(2)], n)
        assert rc == DALEK_NONE and ok == bytes(n) and set(out) == {b32(1)}


def test_torsion_flags(eng, orc, golden):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(10)
    tors = [orc.p3_from_limbs(t["limbs"]) for t in golden["EIGHT_TORSION"]]
    prime = random_points(orc, rnd, 8)
    mixed = [orc.add(P, T) for P, T in zip(prime, tors[1:] + tors[:1])]
    pts = tors + prime + mixed
    want_flags = [1 | (2 if i == 0 else 0) | 4 for i in range(8)] + [6] * 8 + [4] * 7 + [6]
    assert list(eng.torsion_batch(b"".join(orc.compress(P) for P in pts), len(pts))) == want_flags
    ext = b"".join(point_input(orc, P, EXTENDED) for P in pts)
    assert list(eng.torsion_batch(ext, len(pts), EXTENDED)) == want_flags
    assert list(eng.torsion_batch(orc.compress(prime[0]) + b32(2), 2)) == [6, 0]
    encs = [orc.compress(P) for P in pts]
    assert pkg.EdwardsPoint.is_small_order_batch(encs, engine=eng) == [bool(f & 1) for f in want_flags]
    assert pkg.EdwardsPoint.is_torsion_free_batch(encs, engine=eng) == [bool(f & 2) for f in want_flags]
    with pytest.raises(ValueError):
        pkg.EdwardsPoint.is_small_order_batch([b32(2)], engine=eng)


def test_invalid_arguments(eng, orc):
    import ctypes as C
    lib, h = eng.lib, eng.h
    P = orc.compress(orc.basepoint())
    s, top = b32(5), b32(2**255 | 5)
    out = (C.c_uint8 * 64)()
    ok = (C.c_uint8 * 2)()
    mb = lib.dalek_b200_mul_batch
    assert mb(h, top + s, 2, P, COMPRESSED, 1, 2, 0, out, ok) == INVALID        # bit 255 without the clamp flag
    assert mb(h, top + s, 2, P, COMPRESSED, 1, 2, 1, out, ok) == 0              # clamped: accepted
    assert mb(h, s * 3, 3, P, COMPRESSED, 1, 2, 0, out, ok) == INVALID          # n_scalars not 1 or n
    assert mb(h, s, 1, P * 3, COMPRESSED, 3, 2, 0, out, ok) == INVALID          # n_points not 1 or n
    assert mb(h, s, 1, P, COMPRESSED, 0, 2, 0, out, ok) == INVALID
    assert mb(h, s, 1, P, RISTRETTO, 1, 2, 1, out, ok) == INVALID               # clamp with Ristretto
    assert mb(h, s, 1, P, 7, 1, 2, 0, out, ok) == INVALID                       # unknown format
    assert mb(h, s, 1, P, COMPRESSED, 1, 2, 2, out, ok) == INVALID              # unknown flag
    assert mb(h, None, 1, P, COMPRESSED, 1, 2, 0, out, ok) == INVALID
    assert mb(h, s, 1, None, COMPRESSED, 1, 2, 0, out, ok) == INVALID
    assert mb(h, s, 1, P, COMPRESSED, 1, 2, 0, None, ok) == INVALID
    assert mb(h, s, 1, P, COMPRESSED, 1, 2, 0, out, None) == 0                  # ok is nullable
    assert mb(h, None, 0, None, COMPRESSED, 0, 0, 0, None, None) == 0           # n = 0
    d_top, d_p, d_out = dev(top + s), dev(P), dev(bytes(64))
    mbd = lib.dalek_b200_mul_batch_dev
    assert mbd(h, d_top.data_ptr(), 2, d_p.data_ptr(), COMPRESSED, 1, 2, 0, d_out.data_ptr(), None) == INVALID
    assert mbd(h, d_top.data_ptr(), 2, d_p.data_ptr(), COMPRESSED, 1, 2, 1, d_out.data_ptr(), None) == 0
    assert mbd(h, None, 0, None, COMPRESSED, 0, 0, 0, None, None) == 0
    tb = lib.dalek_b200_edwards_torsion_batch
    assert tb(h, P, RISTRETTO, 1, ok) == INVALID
    assert tb(h, None, COMPRESSED, 1, ok) == INVALID
    assert tb(h, None, COMPRESSED, 0, None) == 0


def test_python_wrappers(eng, orc, golden):
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(12)
    a, base = bytes.fromhex(golden["A_SCALAR"]), bytes.fromhex(golden["BASEPOINT"])
    assert pkg.EdwardsPoint.mul_batch(a, base, engine=eng).hex() == golden["A_TIMES_BASEPOINT"]
    pts = random_points(orc, rnd, 3)
    encs = [orc.compress(P) for P in pts]
    ss = [b32(rnd.randrange(L)) for _ in range(3)]
    assert pkg.EdwardsPoint.mul_batch(ss, encs, engine=eng) == [want(orc, s, P, COMPRESSED) for s, P in zip(ss, pts)]
    assert pkg.EdwardsPoint.mul_batch(ss[0], encs, engine=eng) == [want(orc, ss[0], P, COMPRESSED) for P in pts]
    assert pkg.EdwardsPoint.mul_batch(ss, encs[0], engine=eng) == [want(orc, s, pts[0], COMPRESSED) for s in ss]
    raw = [rnd.randbytes(32) for _ in range(3)]
    assert pkg.EdwardsPoint.mul_clamped_batch(raw, encs[1], engine=eng) == [want(orc, r, pts[1], COMPRESSED, True) for r in raw]
    renc = [orc.ristretto_compress(P) for P in pts]
    assert pkg.RistrettoPoint.mul_batch(ss, renc, engine=eng) == [want(orc, s, P, RISTRETTO) for s, P in zip(ss, pts)]
    with pytest.raises(ValueError):
        pkg.EdwardsPoint.mul_batch(ss[0], [encs[0], b32(2)], engine=eng)
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.mul_batch(ss[0], b32(2**255 - 1), engine=eng)


def test_timers_are_set(eng, orc):
    rnd = random.Random(13)
    P = orc.compress(random_points(orc, rnd, 1)[0])
    eng.mul_batch(b32(3) * 2000, 2000, P, 1, 2000)
    assert eng.last_call_ms() > 0 and eng.last_kernel_ms()[0] > 0
