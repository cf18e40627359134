"""The batched group operations on the GPU (csrc/point_ops.cu) against the C oracle: Add / Sub / Neg / double /
mul_by_cofactor for both groups, every input and output format, broadcast operands and piece boundaries, on host and device
buffers; equality semantics; segmented sums against oracle_sum_points and msm_batch with unit scalars; an ElGamal round
trip through engine calls; and the argument checks."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import curve25519_dalek_b200 as pkg
import oracle_lib
import pyref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = pyref.L
COMPRESSED, EXTENDED, RISTRETTO = pkg.POINTS_COMPRESSED, pkg.POINTS_EXTENDED, pkg.POINTS_RISTRETTO
PIECE = 1 << 16
BIG = [PIECE - 1, PIECE + 1, 3 * PIECE + 5]
ID_EDWARDS, ID_RISTRETTO = (1).to_bytes(32, "little"), bytes(32)


def b32(x):
    return x.to_bytes(32, "little")


def limbs_bytes(limbs):
    return b"".join(int(v).to_bytes(8, "little") for v in limbs)


@pytest.fixture(scope="module")
def eng():
    e = pkg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def orc():
    o = oracle_lib.load()
    o.lib.oracle_sum_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    return o


class Pool:
    """Points of one group with their encodings; results of the oracle cached by pool index."""

    def __init__(self, orc, rist, rnd):
        with open(os.path.join(ROOT, "tests", "golden", "scalar_mul.json")) as f:
            tors = [orc.p3_from_limbs(t["limbs"]) for t in json.load(f)["EIGHT_TORSION"]]
        B = orc.basepoint()
        self.orc, self.rist = orc, rist
        pts = [orc.scalarmul(b32(rnd.randrange(L)), B) for _ in range(40)]
        if rist:
            pts = [orc.identity()] + pts
            # representatives: P + T for 4-torsion T are the same Ristretto point
            four = [T for T in tors if orc.is_identity(orc.mul_by_pow_2(T, 2))]
            self.P = [orc.add(P, four[i % 4]) for i, P in enumerate(pts)]
        else:
            self.P = [orc.identity()] + tors + pts + [orc.add(pts[i], tors[i]) for i in range(8)]
        self.enc = [self.encode(P) for P in self.P]
        self.limbs = [limbs_bytes(orc.p3_limbs(P)) for P in self.P]
        self.fmt = RISTRETTO if rist else COMPRESSED
        self.identity = ID_RISTRETTO if rist else ID_EDWARDS
        self.cache = {}

    def encode(self, P):
        return self.orc.ristretto_compress(P) if self.rist else self.orc.compress(P)

    def result(self, op, i, j=0):
        key = (op, i, j)
        if key not in self.cache:
            o, P, Q = self.orc, self.P[i], self.P[j]
            R = {"add": lambda: o.add(P, Q), "sub": lambda: o.sub(P, Q), "neg": lambda: o.sub(o.identity(), P),
                 "double": lambda: o.double(P), "mul_by_cofactor": lambda: o.mul_by_pow_2(P, 3)}[op]()
            self.cache[key] = self.encode(R)
        return self.cache[key]

    def inputs(self, idx, fmt):
        src = self.limbs if fmt == EXTENDED else self.enc
        return b"".join(src[k] for k in idx)


@pytest.fixture(scope="module")
def pools(orc):
    rnd = random.Random(41)
    return {"edwards": Pool(orc, False, rnd), "ristretto": Pool(orc, True, rnd)}


def to_dev(data):
    import torch
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def to_host(t, nbytes):
    return t.cpu().numpy().tobytes()[:nbytes]


def decode_extended(eng, pool, raw, n):
    """EXTENDED results -> the group's encodings, through the oracle (one call per distinct result)."""
    seen, out = {}, []
    for i in range(n):
        lb = raw[160 * i:160 * i + 160]
        if lb not in seen:
            P = pool.orc.p3_from_limbs([int.from_bytes(lb[8 * k:8 * k + 8], "little") for k in range(20)])
            seen[lb] = pool.encode(P)
        out.append(seen[lb])
    return b"".join(out)


def run_binary(eng, pool, op, a_idx, b_idx, in_fmt, out_fmt, dev):
    n = max(len(a_idx), len(b_idx))
    a, b = pool.inputs(a_idx, in_fmt), pool.inputs(b_idx, in_fmt)
    kw = dict(point_fmt=in_fmt, sub=op == "sub", ristretto=pool.rist, out_fmt=out_fmt, want_ok=True)
    if dev:
        rc, out, ok = eng.point_add_batch(to_dev(a), len(a_idx), to_dev(b), len(b_idx), n, device_ptrs=True, **kw)
        size = 160 if out_fmt == EXTENDED else 32
        out, ok = to_host(out, size * n), to_host(ok, n)
    else:
        rc, out, ok = eng.point_add_batch(a, len(a_idx), b, len(b_idx), n, **kw)
    return rc, out, ok


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("out_ext", [False, True], ids=["out_enc", "out_ext"])
@pytest.mark.parametrize("in_ext", [False, True], ids=["in_enc", "in_ext"])
@pytest.mark.parametrize("group", ["edwards", "ristretto"])
def test_add_sub_parity(eng, pools, group, in_ext, out_ext, dev):
    pool = pools[group]
    rnd = random.Random("%s-%d-%d-%d" % (group, in_ext, out_ext, dev))
    in_fmt = EXTENDED if in_ext else pool.fmt
    out_fmt = EXTENDED if out_ext else pool.fmt
    np_ = len(pool.P)
    cases = [(n, n) for n in [1, 7] + BIG] + [(1, 9), (9, 1), (1, PIECE + 1), (3 * PIECE + 5, 1)]
    for op in ("add", "sub"):
        for na, nb in cases:
            n = max(na, nb)
            a_idx = [rnd.randrange(np_) for _ in range(na)]
            b_idx = [rnd.randrange(np_) for _ in range(nb)]
            rc, out, ok = run_binary(eng, pool, op, a_idx, b_idx, in_fmt, out_fmt, dev)
            want = b"".join(pool.result(op, a_idx[i if na > 1 else 0], b_idx[i if nb > 1 else 0]) for i in range(n))
            got = decode_extended(eng, pool, out, n) if out_ext else out
            assert rc == 0 and ok == b"\x01" * n and got == want, (op, na, nb)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("group", ["edwards", "ristretto"])
def test_unary_parity(eng, pools, group, dev):
    pool = pools[group]
    rnd = random.Random(43)
    ops = ["neg", "double"] + (["mul_by_cofactor"] if group == "edwards" else [])
    for op in ops:
        for in_fmt, out_fmt, n in [(pool.fmt, pool.fmt, 3 * PIECE + 5), (EXTENDED, pool.fmt, PIECE + 1), (pool.fmt, EXTENDED, 1000),
                                   (EXTENDED, EXTENDED, PIECE - 1), (pool.fmt, pool.fmt, 1)]:
            idx = [rnd.randrange(len(pool.P)) for _ in range(n)]
            pts = pool.inputs(idx, in_fmt)
            kw = dict(point_fmt=in_fmt, ristretto=pool.rist, out_fmt=out_fmt, want_ok=True)
            if dev:
                rc, out, ok = eng.point_unary_batch(op, to_dev(pts), n, device_ptrs=True, **kw)
                out, ok = to_host(out, (160 if out_fmt == EXTENDED else 32) * n), to_host(ok, n)
            else:
                rc, out, ok = eng.point_unary_batch(op, pts, n, **kw)
            got = decode_extended(eng, pool, out, n) if out_fmt == EXTENDED else out
            assert rc == 0 and ok == b"\x01" * n
            assert got == b"".join(pool.result(op, i) for i in idx), (op, in_fmt, out_fmt, n)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("group", ["edwards", "ristretto"])
def test_undecodable_slots(eng, pools, group, dev):
    pool = pools[group]
    n = 3 * PIECE + 5
    bad_enc = (2).to_bytes(32, "little") if group == "edwards" else b"\xff" * 32
    rnd = random.Random(44)
    a_idx = [rnd.randrange(len(pool.P)) for _ in range(n)]
    a = bytearray(pool.inputs(a_idx, pool.fmt))
    bads = [0, PIECE - 1, PIECE, n - 1]
    for i in bads:
        a[32 * i:32 * i + 32] = bad_enc
    b = pool.enc[3]
    if dev:
        rc, out, ok = eng.point_add_batch(to_dev(bytes(a)), n, to_dev(b), 1, n, point_fmt=pool.fmt, device_ptrs=True, want_ok=True)
        out, ok = to_host(out, 32 * n), to_host(ok, n)
    else:
        rc, out, ok = eng.point_add_batch(bytes(a), n, b, 1, n, point_fmt=pool.fmt, want_ok=True)
    assert rc == 1
    for i in range(n):
        if i in bads:
            assert ok[i] == 0 and out[32 * i:32 * i + 32] == pool.identity
        elif i % 997 == 0:
            assert ok[i] == 1 and out[32 * i:32 * i + 32] == pool.result("add", a_idx[i], 3)
    assert sum(ok) == n - len(bads)
    rc, flags = eng.point_eq_batch(bytes(a), n, None, 0, n, point_fmt=pool.fmt)
    assert rc == 1 and [flags[i] for i in bads] == [0] * 4 and all(flags[i] & 2 for i in range(1, 50))


def test_equality_semantics(eng, orc, pools):
    pool = pools["edwards"]
    tors = pool.P[1:9]
    # is_identity on the eight small-order points: Edwards only the identity, Ristretto the 4-torsion coset
    enc = b"".join(orc.compress(T) for T in tors)
    assert pkg.EdwardsPoint.is_identity_batch([orc.compress(T) for T in tors], engine=eng) == \
        [orc.is_identity(T) for T in tors]
    rc, flags = eng.point_eq_batch(b"".join(limbs_bytes(orc.p3_limbs(T)) for T in tors), 8, None, 0, 8, point_fmt=EXTENDED,
                                   ristretto=True)
    assert rc == 0 and [f & 1 for f in flags] == [int(orc.is_identity(orc.mul_by_pow_2(T, 2))) for T in tors]
    assert pkg.RistrettoPoint.is_identity_batch([ID_RISTRETTO], engine=eng) == [True]
    # Ristretto coset invariance: P + T equals P as a Ristretto point, not as an Edwards point (T 4-torsion, not 0)
    four = [T for T in tors if orc.is_identity(orc.mul_by_pow_2(T, 2)) and not orc.is_identity(T)]
    P = orc.scalarmul(b32(12345), orc.basepoint())
    a = b"".join(limbs_bytes(orc.p3_limbs(orc.add(P, T))) for T in four)
    b = limbs_bytes(orc.p3_limbs(P))
    rc, fr = eng.point_eq_batch(a, 3, b, 1, 3, point_fmt=EXTENDED, ristretto=True)
    rc2, fe = eng.point_eq_batch(a, 3, b, 1, 3, point_fmt=EXTENDED)
    assert rc == rc2 == 0 and list(fr) == [3] * 3 and list(fe) == [2] * 3
    # a non-canonical CompressedEdwardsY equals its canonical form
    nc = bytearray(b32(2**255 - 19 + 1))
    assert pkg.EdwardsPoint.eq_batch(bytes(nc), ID_EDWARDS, engine=eng) is True
    assert pkg.EdwardsPoint.eq_batch([orc.compress(P)] * 2, [orc.compress(P), enc[:32]], engine=eng) == [True, False]
    # parity against the oracle at a piece boundary, with broadcast
    for g in ("edwards", "ristretto"):
        pool = pools[g]
        rnd = random.Random(45)
        n = PIECE + 1
        a_idx = [rnd.randrange(len(pool.P)) for _ in range(n)]
        rc, flags = eng.point_eq_batch(pool.inputs(a_idx, EXTENDED), n, pool.limbs[5], 1, n, point_fmt=EXTENDED, ristretto=pool.rist)
        eq = orc.ristretto_ct_eq if pool.rist else orc.ct_eq
        want = {k: eq(pool.P[k], pool.P[5]) for k in set(a_idx)}
        assert rc == 0 and all(flags[i] == 2 | int(want[a_idx[i]]) for i in range(n))


def oracle_sum(orc, pool, idx):
    arr = (oracle_lib.P3 * max(1, len(idx)))()
    for k, i in enumerate(idx):
        arr[k] = pool.P[i]
    out = (C.c_uint8 * 32)()
    orc.lib.oracle_sum_points(out, None, arr, len(idx))
    if pool.rist:
        R = orc.identity()
        for i in idx:
            R = orc.add(R, pool.P[i])
        return orc.ristretto_compress(R)
    return bytes(out)


def counted_sum(orc, pool, idx):
    """The sum as sum_k count_k P_k (for segments too long to add one by one in Python)."""
    R = orc.identity()
    for k, c in zip(*np.unique(np.array(idx), return_counts=True)):
        R = orc.add(R, orc.scalarmul(b32(int(c)), pool.P[int(k)]))
    return pool.encode(R)


def run_sum(eng, pool, idx, sizes, in_fmt, out_fmt, dev):
    offs = np.zeros(len(sizes) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(sizes)
    pts = pool.inputs(idx, in_fmt) or b"\0"
    m = len(sizes)
    kw = dict(point_fmt=in_fmt, ristretto=pool.rist, out_fmt=out_fmt, want_ok=True)
    if dev:
        rc, out, ok = eng.point_sum_batch(to_dev(pts), to_dev(offs.tobytes()), m, device_ptrs=True, **kw)
        out, ok = to_host(out, (160 if out_fmt == EXTENDED else 32) * m), to_host(ok, m)
    else:
        rc, out, ok = eng.point_sum_batch(pts, offs, m, **kw)
    if out_fmt == EXTENDED:
        out = decode_extended(eng, pool, out, m)
    return rc, out, ok


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("group", ["edwards", "ristretto"])
def test_sum_segment_lengths(eng, orc, pools, group, dev):
    pool = pools[group]
    rnd = random.Random(46)
    sizes = [0, 1, 2, 31, 32, 33, 1023, 1024, 1025, 2049, 0, 5, (1 << 20) + 3]
    idx = [rnd.randrange(len(pool.P)) for _ in range(sum(sizes))]
    segs, at = [], 0
    for s in sizes:
        segs.append(idx[at:at + s]); at += s
    want = b"".join(oracle_sum(orc, pool, s) if len(s) < 5000 else counted_sum(orc, pool, s) for s in segs)
    for in_fmt, out_fmt in [(pool.fmt, pool.fmt), (EXTENDED, EXTENDED)]:
        rc, out, ok = run_sum(eng, pool, idx, sizes, in_fmt, out_fmt, dev)
        assert rc == 0 and ok == b"\x01" * len(sizes) and out == want, (in_fmt, out_fmt)


def test_many_small_sums_and_msm_batch(eng, orc, pools):
    for g in ("edwards", "ristretto"):
        pool = pools[g]
        rnd = random.Random(47)
        m, k = 1 << 16, 4
        idx = [rnd.randrange(len(pool.P)) for _ in range(m * k)]
        rc, out, ok = run_sum(eng, pool, idx, [k] * m, pool.fmt, pool.fmt, False)
        assert rc == 0 and ok == b"\x01" * m
        for j in range(0, m, 1031):
            assert out[32 * j:32 * j + 32] == oracle_sum(orc, pool, idx[k * j:k * j + k])
        offs = np.arange(0, m * k + 1, k, dtype=np.uint64)
        rc2, want, ok2, _ = eng.msm_batch(b32(1) * (m * k), pool.inputs(idx, pool.fmt), offs, m, point_fmt=pool.fmt)
        assert rc2 == 0 and out == want


@pytest.mark.parametrize("group", ["edwards", "ristretto"])
def test_sum_with_an_undecodable_point(eng, orc, pools, group):
    pool = pools[group]
    sizes = [3, 2000, 7, 0, PIECE + 9]
    rnd = random.Random(48)
    idx = [rnd.randrange(len(pool.P)) for _ in range(sum(sizes))]
    pts = bytearray(pool.inputs(idx, pool.fmt))
    bad = 3 + 1500
    pts[32 * bad:32 * bad + 32] = (2).to_bytes(32, "little") if group == "edwards" else b"\xff" * 32
    offs = np.zeros(len(sizes) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(sizes)
    rc, out, ok = eng.point_sum_batch(bytes(pts), offs, len(sizes), point_fmt=pool.fmt, want_ok=True)
    assert rc == 1 and list(ok) == [1, 0, 1, 1, 1]
    assert out[32:64] == pool.identity and out[96:128] == pool.identity
    assert out[:32] == oracle_sum(orc, pool, idx[:3]) and out[64:96] == oracle_sum(orc, pool, idx[2003:2010])
    with pytest.raises(ValueError):
        (pkg.EdwardsPoint if group == "edwards" else pkg.RistrettoPoint).sum([bytes(pts[32 * bad:32 * bad + 32])], engine=eng)


def test_elgamal_round_trip(eng, orc):
    rnd = random.Random(49)
    R = pkg.RistrettoPoint
    n = 1 << 16
    x = b32(rnd.randrange(1, L))
    Pk = R.mul_base_batch(x, engine=eng)
    payloads = [rnd.randbytes(16) for _ in range(n)]
    rs = [b32(rnd.randrange(1, L)) for _ in range(n)]
    C1 = R.mul_base_batch(rs, engine=eng)
    M = R.lizard_encode_batch(payloads, engine=eng)
    C2 = R.add_batch(M, R.mul_batch(rs, Pk, engine=eng), engine=eng)
    back = R.lizard_decode_batch(R.sub_batch(C2, R.mul_batch(x, C1, engine=eng), engine=eng), engine=eng)
    assert back == payloads
    # homomorphic: the sum of encryptions of m_i B decrypts to (sum m_i) B
    k = 64
    ms = [rnd.randrange(1000) for _ in range(k)]
    c1 = R.mul_base_batch(rs[:k], engine=eng)
    c2 = R.add_batch(R.mul_base_batch([b32(v) for v in ms], engine=eng), R.mul_batch(rs[:k], Pk, engine=eng), engine=eng)
    S1, S2 = R.sum_batch([c1, c2], engine=eng)
    dec = R.sub_batch(S2, R.mul_batch(x, S1, engine=eng), engine=eng)
    assert dec == R.mul_base_batch(b32(sum(ms)), engine=eng)
    assert R.eq_batch(dec, orc.ristretto_compress(orc.scalarmul(b32(sum(ms)), orc.basepoint())), engine=eng) is True


def test_class_surface(eng, orc):
    E = pkg.EdwardsPoint
    B = orc.compress(orc.basepoint())
    two = orc.compress(orc.double(orc.basepoint()))
    assert E.add_batch(B, B, engine=eng) == E.double_batch(B, engine=eng) == two
    assert E.sub_batch(two, B, engine=eng) == B
    assert E.add_batch(B, E.neg_batch(B, engine=eng), engine=eng) == ID_EDWARDS
    assert E.mul_by_cofactor_batch([B], engine=eng) == [orc.compress(orc.mul_by_pow_2(orc.basepoint(), 3))]
    assert E.sum([], engine=eng) == ID_EDWARDS and E.sum([B, B], engine=eng) == two
    assert E.sum_batch([[], [B], [B, B]], engine=eng) == [ID_EDWARDS, B, two]
    with pytest.raises(ValueError):
        E.add_batch(B, (2).to_bytes(32, "little"), engine=eng)
    assert not hasattr(pkg.RistrettoPoint, "mul_by_cofactor_batch")


def test_invalid_arguments_fail_before_device_work(eng):
    lib, h = eng.lib, eng.h
    pt = bytes(32)
    out = (C.c_uint8 * 1024)()
    offs = np.array([0, 2, 1], dtype=np.uint64)
    before = eng.launch_count()
    calls = [
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, COMPRESSED, 2, 0, RISTRETTO, out, None),     # wrong out_fmt
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, RISTRETTO, 2, 0, COMPRESSED, out, None),
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, COMPRESSED, 2, 2, COMPRESSED, out, None),    # RISTRETTO flag
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, COMPRESSED, 2, 4, COMPRESSED, out, None),    # unknown flag
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, 3, 2, 0, 3, out, None),                      # Montgomery
        lambda: lib.dalek_b200_point_add_batch(h, pt, 2, pt, 3, COMPRESSED, 4, 0, COMPRESSED, out, None),    # counts
        lambda: lib.dalek_b200_point_add_batch(h, None, 1, pt, 1, COMPRESSED, 1, 0, COMPRESSED, out, None),  # NULL
        lambda: lib.dalek_b200_point_add_batch(h, pt, 1, pt, 1, COMPRESSED, 1, 0, COMPRESSED, None, None),
        lambda: lib.dalek_b200_point_add_batch_dev(h, None, 1, None, 1, COMPRESSED, 1, 0, COMPRESSED, None, None),
        lambda: lib.dalek_b200_point_unary_batch(h, 3, pt, COMPRESSED, 1, 0, COMPRESSED, out, None),         # bad op
        lambda: lib.dalek_b200_point_unary_batch(h, 2, pt, RISTRETTO, 1, 0, RISTRETTO, out, None),           # cofactor
        lambda: lib.dalek_b200_point_unary_batch(h, 2, pt, EXTENDED, 1, 2, EXTENDED, out, None),
        lambda: lib.dalek_b200_point_unary_batch(h, 0, pt, COMPRESSED, 1, 1, COMPRESSED, out, None),         # SUB flag
        lambda: lib.dalek_b200_point_unary_batch_dev(h, -1, pt, COMPRESSED, 1, 0, COMPRESSED, out, None),
        lambda: lib.dalek_b200_point_eq_batch(h, pt, 1, pt, 1, COMPRESSED, 1, 1, out),                      # SUB flag
        lambda: lib.dalek_b200_point_eq_batch(h, pt, 1, pt, 1, COMPRESSED, 1, 2, out),
        lambda: lib.dalek_b200_point_eq_batch(h, pt, 2, pt, 1, COMPRESSED, 3, 0, out),
        lambda: lib.dalek_b200_point_eq_batch(h, None, 1, pt, 1, COMPRESSED, 1, 0, out),
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 0, offs.ctypes.data, 2, COMPRESSED, out, None),  # decreasing
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 0, np.array([1, 2], dtype=np.uint64).ctypes.data, 1,
                                               COMPRESSED, out, None),                                        # offsets[0] != 0
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 0, np.array([0, 1 << 31], dtype=np.uint64).ctypes.data, 1,
                                               COMPRESSED, out, None),                                        # total >= 2^31
        lambda: lib.dalek_b200_point_sum_batch(h, None, COMPRESSED, 0, np.array([0, 1], dtype=np.uint64).ctypes.data, 1,
                                               COMPRESSED, out, None),
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 0, None, 1, COMPRESSED, out, None),
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 0, np.array([0, 1], dtype=np.uint64).ctypes.data, 1,
                                               RISTRETTO, out, None),
        lambda: lib.dalek_b200_point_sum_batch(h, pt, COMPRESSED, 1, np.array([0, 1], dtype=np.uint64).ctypes.data, 1,
                                               COMPRESSED, out, None),
    ]
    for k, f in enumerate(calls):
        assert f() == -1, k
    assert eng.launch_count() == before
    # n = 0 and m = 0 are no-ops, even with NULL buffers
    assert lib.dalek_b200_point_add_batch(h, None, 0, None, 0, COMPRESSED, 0, 0, COMPRESSED, None, None) == 0
    assert lib.dalek_b200_point_sum_batch(h, None, COMPRESSED, 0, None, 0, COMPRESSED, None, None) == 0
