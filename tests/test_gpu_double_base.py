"""GPU variable-time double-base scalar multiplication: dalek_b200_vartime_double_base_batch / _dev
(EdwardsPoint / RistrettoPoint ::vartime_double_scalar_mul_basepoint, out[i] = a_i A_i + b_i B) against the reference's
KAT, the C oracle (tests/host/double_base_oracle.c), batched two-term MSMs, fixed-base multiplication and the Ed25519
verifier."""
import ctypes as C
import hashlib
import json
import os
import random

import pytest

import double_base_oracle
import oracle_lib
import pyref
from torsion_cases import torsion_points

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L
PRIME = 2**255 - 19
COMPRESSED, EXTENDED, RISTRETTO = 0, 1, 2
DALEK_NONE, INVALID = 1, -1
PIECE = 1 << 16
THREADS = os.cpu_count() or 1


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
def dbo():
    return double_base_oracle.load()


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "kat.json")) as f:
        return json.load(f)["edwards"]


def b32(x):
    return x.to_bytes(32, "little")


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def dev(buf):
    import torch
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()


def run(eng, ab, pts, fmt=COMPRESSED, device=False):
    """(rc, outputs, ok) through host or device buffers; ab: list of 64-byte pairs, pts: list of point inputs"""
    n = len(ab)
    if device:
        rc, out, ok = eng.vartime_double_base_batch(dev(b"".join(ab)), dev(b"".join(pts)), n, fmt, device_ptrs=True, want_ok=True)
        return rc, split(bytes(out.cpu().numpy())[:32 * n]), bytes(ok.cpu().numpy())[:n]
    rc, out, ok = eng.vartime_double_base_batch(b"".join(ab), b"".join(pts), n, fmt, want_ok=True)
    return rc, split(out), ok


def oracle(dbo, ab, pts, fmt=COMPRESSED):
    rc, out, ok = dbo.batch(b"".join(ab), b"".join(pts), len(ab), fmt, THREADS)
    return rc, split(out), ok


def point_input(orc, P, fmt):
    if fmt == EXTENDED:
        return b"".join(int(v).to_bytes(8, "little") for v in orc.p3_limbs(P))
    return orc.ristretto_compress(P) if fmt == RISTRETTO else orc.compress(P)


def random_points(orc, rnd, k):
    B = orc.basepoint()
    return [orc.scalarmul(b32(rnd.randrange(1, L)), B) for _ in range(k)]


def rand_pair(rnd):
    return b32(rnd.randrange(2**255)) + b32(rnd.randrange(2**255))


def edge_scalars():
    return [b32(0), b32(1), b32(L - 1), b32(L), b32(L + 1), b32(2**255 - 1), b32(2**252), bytes([0x88] * 31 + [0x08]),
            bytes([0x88] * 31 + [0x78]), bytes([0x77] * 32), bytes([0xff] * 31 + [0x0f]), bytes([0xff] * 31 + [0x7f]),
            bytes([0x08] * 32), bytes([0xf8] * 31 + [0x7f])]


@pytest.mark.parametrize("device", [False, True])
def test_kat_through_c_abi(eng, kat, device):
    a, b = bytes.fromhex(kat["A_SCALAR"]["hex"]), bytes.fromhex(kat["B_SCALAR"]["hex"])
    A = bytes.fromhex(kat["A_TIMES_BASEPOINT"]["hex"])
    rc, out, ok = run(eng, [a + b], [A], device=device)
    assert rc == 0 and ok == b"\x01" and out == [bytes.fromhex(kat["DOUBLE_SCALAR_MULT_RESULT"]["hex"])]


def test_python_wrappers(eng, orc, dbo, kat):
    import curve25519_dalek_b200 as pkg
    a, b = bytes.fromhex(kat["A_SCALAR"]["hex"]), bytes.fromhex(kat["B_SCALAR"]["hex"])
    A = bytes.fromhex(kat["A_TIMES_BASEPOINT"]["hex"])
    res = bytes.fromhex(kat["DOUBLE_SCALAR_MULT_RESULT"]["hex"])
    assert pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch([a, b], [A, A], [b, a], engine=eng) == \
        [res, dbo.one(b, A, a)[0]]
    rnd = random.Random(31)
    renc = [orc.ristretto_compress(P) for P in random_points(orc, rnd, 3)]
    as_, bs = [b32(rnd.randrange(L)) for _ in range(3)], [b32(rnd.randrange(2**255)) for _ in range(3)]
    assert pkg.RistrettoPoint.vartime_double_scalar_mul_basepoint_batch(as_, renc, bs, engine=eng) == \
        [dbo.one(x, p, y, RISTRETTO)[0] for x, p, y in zip(as_, renc, bs)]
    assert pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch([], [], [], engine=eng) == []
    with pytest.raises(ValueError):
        pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch([a, a], [A, b32(2)], [b, b], engine=eng)
    with pytest.raises(ValueError):
        pkg.RistrettoPoint.vartime_double_scalar_mul_basepoint_batch([a], [b32(2**255 - 1)], [b], engine=eng)
    with pytest.raises(ValueError):
        pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch([b32(2**255)], [A], [b], engine=eng)
    with pytest.raises(ValueError):
        pkg.EdwardsPoint.vartime_double_scalar_mul_basepoint_batch([a], [A, A], [b], engine=eng)


@pytest.mark.parametrize("fmt", [COMPRESSED, EXTENDED, RISTRETTO])
@pytest.mark.parametrize("n", [1, 7, 1000])
def test_oracle_parity(eng, orc, dbo, fmt, n):
    rnd = random.Random(n * 10 + fmt)
    pts = [point_input(orc, P, fmt) for P in random_points(orc, rnd, n)]
    ab = [rand_pair(rnd) for _ in range(n)]
    want = oracle(dbo, ab, pts, fmt)
    assert want[0] == 0
    for device in (False, True):
        assert run(eng, ab, pts, fmt, device) == want, device


@pytest.mark.parametrize("fmt", [COMPRESSED, EXTENDED, RISTRETTO])
def test_piece_boundary(eng, orc, dbo, fmt):
    n = 2 * PIECE + 1                            # three pieces, the last of one item
    rnd = random.Random(40 + fmt)
    pool = [point_input(orc, P, fmt) for P in random_points(orc, rnd, 256)]
    pts = [pool[rnd.randrange(256)] for _ in range(n)]
    ab = [rand_pair(rnd) for _ in range(n)]
    want = oracle(dbo, ab, pts, fmt)
    for device in (False, True):
        assert run(eng, ab, pts, fmt, device) == want, device


def test_edge_scalars_and_special_points(eng, orc, dbo):
    rnd = random.Random(32)
    B = orc.basepoint()
    tors = torsion_points(orc)
    pts = [orc.identity(), B] + list(tors) + [orc.add(P, T) for P, T in zip(random_points(orc, rnd, 8), tors)]
    pts += random_points(orc, rnd, 4)
    r = b32(rnd.randrange(L))
    pairs = [s + r for s in edge_scalars()] + [r + s for s in edge_scalars()] + [s + s for s in edge_scalars()]
    ab = [x for _ in pts for x in pairs]
    for fmt in (COMPRESSED, EXTENDED):
        pin = [point_input(orc, P, fmt) for P in pts for _ in pairs]
        want = oracle(dbo, ab, pin, fmt)
        assert want[0] == 0
        for device in (False, True):
            assert run(eng, ab, pin, fmt, device) == want, (fmt, device)


def test_unreduced_scalars_on_torsion_points(eng, orc, dbo):
    rnd = random.Random(33)
    tors = torsion_points(orc)
    pts, ab = [], []
    for T in tors[1:]:
        P = orc.add(random_points(orc, rnd, 1)[0], T)
        for a in (L, L + 1, 2**255 - 1, rnd.randrange(L, 2**255)):
            pts.append(orc.compress(P))
            ab.append(b32(a) + b32(rnd.randrange(2**255)))
    rc, out, ok = run(eng, ab, pts)
    assert (rc, out, ok) == oracle(dbo, ab, pts)
    reduced = oracle(dbo, [b32(int.from_bytes(x[:32], "little") % L) + x[32:] for x in ab], pts)[1]
    assert sum(o != r for o, r in zip(out, reduced)) >= len(ab) // 2


def test_extended_input_with_random_z(eng, orc, dbo):
    rnd = random.Random(34)
    n = 200
    Ps = random_points(orc, rnd, n)
    pts = []
    for P in Ps:
        x, y = [int.from_bytes(orc.fe_to_bytes(c), "little") for c in (P.X, P.Y)]
        zi = pow(int.from_bytes(orc.fe_to_bytes(P.Z), "little"), PRIME - 2, PRIME)
        x, y = x * zi % PRIME, y * zi % PRIME
        lam = rnd.randrange(1, PRIME)
        coords = [lam * x % PRIME, lam * y % PRIME, lam, lam * x * y % PRIME]
        pts.append(b"".join(((c >> (51 * k)) & (2**51 - 1)).to_bytes(8, "little") for c in coords for k in range(5)))
    ab = [rand_pair(rnd) for _ in range(n)]
    want = oracle(dbo, ab, [orc.compress(P) for P in Ps])
    for device in (False, True):
        assert run(eng, ab, pts, EXTENDED, device) == want


def test_ristretto_coset_invariance(eng, orc):
    rnd = random.Random(35)
    tors = torsion_points(orc)
    four = [orc.identity(), tors[1], tors[3], tors[5]]          # the 4-torsion: orders 1, 4, 2, 4
    for P in random_points(orc, rnd, 5):
        encs = [orc.ristretto_compress(orc.add(P, T)) for T in four]
        assert len(set(encs)) == 1
        x = rand_pair(rnd)
        rc, out, _ = run(eng, [x] * 4, encs, RISTRETTO)
        assert rc == 0 and len(set(out)) == 1
        # the extended coordinates of P + T are four representatives of one Ristretto point
        rc, out_e, _ = run(eng, [x] * 4, [point_input(orc, orc.add(P, T), EXTENDED) for T in four], EXTENDED)
        assert rc == 0
        assert [orc.ristretto_compress(orc.decompress(o)) for o in out_e] == [out[0]] * 4


def test_ristretto_rejection_classes(eng, orc, dbo):
    with open(os.path.join(ROOT, "tests", "golden", "ristretto.json")) as f:
        classes = json.load(f)["classes"]
    rnd = random.Random(36)
    good = [orc.ristretto_compress(P) for P in random_points(orc, rnd, 2)]
    for cls in ("noncanonical", "negative", "nonsquare", "t_negative", "y_zero"):
        for v in classes[cls]:
            encs = [good[0], bytes.fromhex(v["s"]), good[1]]         # neighbours on both sides
            ab = [rand_pair(rnd) for _ in range(3)]
            for device in (False, True):
                rc, out, ok = run(eng, ab, encs, RISTRETTO, device)
                assert rc == DALEK_NONE and ok == b"\x01\x00\x01", (cls, device)
                assert out[1] == bytes(32)
                assert [out[0], out[2]] == [dbo.one(ab[i][:32], encs[i], ab[i][32:], RISTRETTO)[0] for i in (0, 2)]


def test_undecodable_edwards_points(eng, orc, dbo):
    rnd = random.Random(37)
    encs = [orc.compress(P) for P in random_points(orc, rnd, 6)]
    encs[2] = encs[4] = b32(2)                                        # y = 2 is not on the curve
    ab = [rand_pair(rnd) for _ in range(6)]
    want = oracle(dbo, ab, encs)
    assert want[0] == 1 and want[2] == bytes([1, 1, 0, 1, 0, 1])
    for device in (False, True):
        assert run(eng, ab, encs, COMPRESSED, device) == (DALEK_NONE, want[1], want[2])
        assert run(eng, ab, encs, COMPRESSED, device)[1][2] == b32(1)


@pytest.mark.parametrize("fmt", [COMPRESSED, RISTRETTO])
def test_equals_two_term_msm_batch(eng, orc, fmt):
    import numpy as np
    n = 1 << 16
    rnd = random.Random(38 + fmt)
    pool = [point_input(orc, P, fmt) for P in random_points(orc, rnd, 256)]
    Bin = point_input(orc, orc.basepoint(), fmt)
    pts = [pool[rnd.randrange(256)] for _ in range(n)]
    ab = [b32(rnd.randrange(L)) + b32(rnd.randrange(L)) for _ in range(n)]
    rc, out, ok = run(eng, ab, pts, fmt)
    assert rc == 0 and ok == b"\x01" * n
    offs = np.arange(0, 2 * n + 1, 2, dtype=np.uint64)
    rc2, msm, ok2, _ = eng.msm_batch(b"".join(ab), b"".join(p + Bin for p in pts), offs, n, point_fmt=fmt)
    assert rc2 == 0 and ok2 == b"\x01" * n
    assert out == split(msm)


def test_two_to_the_twenty_against_fixed_base(eng):
    """A_i = t_i B: every output equals mul_base((a_i t_i + b_i) mod l)"""
    n = 1 << 20
    rnd = random.Random(39)
    ts = [rnd.randrange(1, L) for _ in range(n)]
    _, A = eng.mul_base_batch(b"".join(b32(t) for t in ts), n)
    as_ = [rnd.randrange(2**255) for _ in range(n)]
    bs = [rnd.randrange(2**255) for _ in range(n)]
    rc, out, ok = eng.vartime_double_base_batch(b"".join(b32(a) + b32(b) for a, b in zip(as_, bs)), A, n, want_ok=True)
    assert rc == 0 and ok == b"\x01" * n
    _, want = eng.mul_base_batch(b"".join(b32((a * t + b) % L) for a, t, b in zip(as_, ts, bs)), n)
    assert out == want


def test_ed25519_testvectors_match_verify_each(eng):
    with open(os.path.join(ROOT, "tests", "golden", "ed25519_testvectors.json")) as f:
        tv = json.load(f)["vectors"]
    H = bytes.fromhex
    msgs = [H(v["msg"]) for v in tv]
    sigs = [H(v["sig"]) for v in tv]
    keys = [H(v["pk"]) for v in tv]
    for i in range(0, len(tv), 9):                                  # some failures too
        msgs[i] += b"x"
    ab, negA = [], []
    for m, s, k in zip(msgs, sigs, keys):
        h = int.from_bytes(hashlib.sha512(s[:32] + k + m).digest(), "little") % L
        ab.append(b32(h) + s[32:])
        negA.append(k[:31] + bytes([k[31] ^ 0x80]))                 # -A: the sign bit of x flipped
    rc, out, ok = run(eng, ab, negA)
    assert ok == b"\x01" * len(tv)
    offs = [0]
    for m in msgs:
        offs.append(offs[-1] + len(m))
    import numpy as np
    flat = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy()
    _, verdicts = eng.verify_each_flat(flat, np.array(offs, dtype=np.uint64), b"".join(sigs), b"".join(keys), len(tv))
    mine = [0 if o == s[:32] else 1 for o, s in zip(out, sigs)]
    assert mine == [0 if v == 0 else 1 for v in verdicts]
    assert 0 < sum(mine) < len(tv)


def test_invalid_arguments(eng, orc):
    lib, h = eng.lib, eng.h
    P = orc.compress(orc.basepoint())
    x, top = b32(5) + b32(7), b32(5) + b32(2**255 | 7)
    out = (C.c_uint8 * 64)()
    ok = (C.c_uint8 * 2)()
    f = lib.dalek_b200_vartime_double_base_batch
    launches = eng.launch_count()
    assert f(h, top + x, P * 2, COMPRESSED, 2, out, ok) == INVALID              # bit 255 of b: nothing launched
    assert f(h, b32(2**255) + b32(1) + x, P * 2, COMPRESSED, 2, out, ok) == INVALID   # bit 255 of a
    assert eng.launch_count() == launches
    assert f(h, x * 2, P * 2, 3, 2, out, ok) == INVALID                         # unknown format
    assert f(h, x * 2, P * 2, -1, 2, out, ok) == INVALID
    assert f(h, None, P * 2, COMPRESSED, 2, out, ok) == INVALID
    assert f(h, x * 2, None, COMPRESSED, 2, out, ok) == INVALID
    assert f(h, x * 2, P * 2, COMPRESSED, 2, None, ok) == INVALID
    assert f(h, None, None, COMPRESSED, 0, None, None) == 0                     # n = 0
    assert eng.launch_count() == launches
    assert f(h, x * 2, P * 2, COMPRESSED, 2, out, None) == 0                   # ok is nullable
    assert eng.launch_count() > launches
    fd = lib.dalek_b200_vartime_double_base_batch_dev
    d_top, d_p, d_out = dev(top + x), dev(P * 2), dev(bytes(64))
    launches = eng.launch_count()
    assert fd(h, d_top.data_ptr(), d_p.data_ptr(), COMPRESSED, 2, d_out.data_ptr(), None) == INVALID   # after the batch ran
    assert eng.launch_count() > launches
    d_x = dev(x * 2)
    assert fd(h, d_x.data_ptr(), d_p.data_ptr(), COMPRESSED, 2, d_out.data_ptr(), None) == 0
    assert fd(h, d_x.data_ptr(), d_p.data_ptr(), 3, 2, d_out.data_ptr(), None) == INVALID
    assert fd(h, None, d_p.data_ptr(), COMPRESSED, 2, d_out.data_ptr(), None) == INVALID
    assert fd(h, None, None, COMPRESSED, 0, None, None) == 0


def test_timers_and_launch_count(eng, orc):
    rnd = random.Random(41)
    P = orc.compress(random_points(orc, rnd, 1)[0])
    for device in (False, True):
        before = eng.launch_count()
        rc, _, _ = run(eng, [rand_pair(rnd) for _ in range(3000)], [P] * 3000, COMPRESSED, device)
        assert rc == 0 and eng.launch_count() > before
        assert eng.last_call_ms() > 0 and eng.last_kernel_ms()[0] > 0
