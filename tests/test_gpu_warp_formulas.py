"""Device-level parity of the point code that runs every MSM's chain of dependent point operations, against exact integer
formulas mod p = 2^255 - 19:

  * csrc/warp4.cuh      the 4-lane integer point code of k_plain_sum and k_heavy_fixup;
  * csrc/warp4_f64.cuh  the 4-lane and 20-lane FP64 point code of k_combine, k_chunk_reduce, k_finish_windows, the
                        inversion of k_prep_invert and the vartime Straus loop;
  * csrc/ge64.cuh       the bucket kernel's mixed additions, ge64_dbl and ge64_add_p3;
  * csrc/fe64.cuh, x25519.cuh  the FP64 exponentiation chains of decompression, Elligator and X25519.

A TEST-ONLY library (tests/device/warp_device_check.cu, compiled from the product headers) runs each operation on free
field elements -- coordinates that are not points on the curve -- so every limb can sit at the bound the headers state,
and returns the raw output limbs of every lane.  The model below is the reference's formulas
(curve25519-dalek/src/backend/serial/curve_models.rs:365-372 completed -> extended, :381-397 doubling, :411-494
projective- and affine-Niels addition and subtraction; src/edwards.rs:528-535 as_projective_niels), and every output
coordinate is compared mod p, so a formula that is right only on the curve, or a lane that plays the wrong role, fails.
The device formulas are the same polynomials as the reference's, so no comparison needs on-curve inputs except the
end-to-end ones at the bottom, which check whole sums against the C oracle.  A device build has no assertions: the
limb bounds are asserted here on the raw limbs."""
import ctypes as C
import math
import os
import random
import sys

import numpy as np
import pytest

import pyref
from test_w4_host import w4  # noqa: F401  (the emulated warp of tests/host/w4_host_check.cpp)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**255 - 19
D = -121665 * pow(121666, P - 2, P) % P
D2 = 2 * D % P
SH25 = [0, 26, 51, 77, 102, 128, 153, 179, 204, 230]
M25 = [(1 << (25 if i & 1 else 26)) - 1 for i in range(10)]
FIXED = (0, 1, 19, P - 1, P, 2**255 - 20, 2**255 - 1)
NMODES = 6                                     # random, all +bound, all -bound, alternating, one non-zero limb, fixed
NPT = 1 << 14                                  # items per point formula

# Balanced FP64 limbs of scale 1, with the slack of fe64_finish (outputs of fe64_mul) and of the 20-lane carry
B10, B14 = (1 << 50) + (1 << 10), (1 << 50) + (1 << 14)
B15 = (1 << 50) + (1 << 15)                     # what w20_mul and the 20-lane point code may leave
# Largest limbs fe_carry64 can leave: 26 / 25 bits, except limb 1, which takes the last carry out of limb 0 after the
# x19 wrap of a 64-bit column 9:  ((2^26 - 1) + 19 (2^39 - 1)) >> 26 = 19 * 2^13
FE_MAX = [m for m in M25]
FE_MAX[1] += 19 << 13
FE_LIM = [1.01 * (1 << (25 if i & 1 else 26)) for i in range(10)]   # scale 1 of fe.cuh

W20_MUL, W20_SQ, W20_CARRY, W20_SQN, W20_INVERT = range(5)
CH_POW22501, CH_POW_P58, CH_INVERT_F64, CH_X25519_INVERT, CH_FROMBYTES, CH_CSWAP, CH_CMOV = range(7)
GE_MADD, GE_PADD, GE_DBL, GE_DBL_NO_T, GE_ADD_P3 = range(5)
W4_ADD, W4_SHFL, W4_FIXUP = range(3)
W4F_DBL, W4F_ADD, W4F_PADD, W4F_SHFL = range(4)
W20_DBL, W20_ADD, W20_LOAD_STORE = range(3)


@pytest.fixture(scope="module")
def dev():
    sys.path.insert(0, os.path.join(ROOT, "tests", "device"))
    import build as devbuild
    lib = C.CDLL(devbuild.build("warp_device_check"))
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.w20_field_check.argtypes = [i, sz, vp, vp, i, vp]
    lib.chain_check.argtypes = [i, sz, vp, vp]
    lib.ge64_check.argtypes = [i, sz, vp, vp]
    lib.w4_check.argtypes = [i, sz, vp, sz, i, i, vp, vp]
    lib.w4f_check.argtypes = [i, sz, vp, sz, i, vp]
    lib.w20_point_check.argtypes = [i, sz, vp, vp, vp, vp]
    lib.combine_check.argtypes = [vp, i, i, i, vp, vp, vp]
    return lib


def ptr(a):
    return a.ctypes.data if a is not None else None


# ---- values ----------------------------------------------------------------------------------------------------------
def vals51(a):
    """Integer values of rows of five radix-2^51 limbs (not reduced)."""
    return [x0 + (x1 << 51) + (x2 << 102) + (x3 << 153) + (x4 << 204) for x0, x1, x2, x3, x4 in a.tolist()]


def vals25(a):
    return [sum(x << s for x, s in zip(row, SH25)) for row in a.tolist()]


def coords51(a):
    """(n, 20) limbs -> four lists of coordinate values mod p."""
    return [[v % P for v in vals51(a[:, 5 * k:5 * k + 5])] for k in range(4)]


def coords25(a):
    return [[v % P for v in vals25(a[:, 10 * k:10 * k + 10])] for k in range(4)]


def balanced(v):
    """Balanced radix-2^51 limbs of v < 2^256 (the carry out of the top limb wraps as 19)."""
    out = []
    for _ in range(5):
        l = v & ((1 << 51) - 1)
        if l >= 1 << 50:
            l -= 1 << 51
        out.append(l)
        v = (v - l) >> 51
    out[0] += 19 * v
    return out


FIXED51 = np.array([balanced(v) for v in FIXED], dtype=np.int64)
FIXED25 = np.array([[(v >> s) & m for s, m in zip(SH25, M25)] for v in FIXED], dtype=np.int64)
FIXEDU51 = np.array([[(v >> (51 * k)) & ((1 << 51) - 1) for k in range(5)] for v in FIXED], dtype=np.int64)


def modes(rng, n, ncoord):
    """Operand mode per item and coordinate: the first half of the items use one mode for all their coordinates (every
    mode in turn), the second half draw each coordinate's mode."""
    m = rng.integers(0, NMODES, size=(n, ncoord))
    m[:n // 2] = (np.arange(n // 2) % NMODES)[:, None]
    return m


def _by_mode(rng, mode, lo, hi, fixed):
    """Rows of limbs in [lo, hi] (per limb) chosen by mode: random, all hi, all lo, alternating hi / lo, one limb at hi
    (or lo when lo < 0), a fixed value."""
    n, w = len(mode), len(hi)
    hi = np.asarray(hi, dtype=np.int64)[None, :]
    lo = np.asarray(lo, dtype=np.int64)[None, :]
    out = (lo + np.floor(rng.random((n, w)) * (hi - lo + 1).astype(np.float64)).astype(np.int64))
    out = np.minimum(out, hi)
    flip = rng.random((n, 1)) < 0.5
    alt = np.where((np.arange(w)[None, :] % 2 == 0) ^ flip, hi, lo)
    one = np.zeros((n, w), dtype=np.int64)
    pos = rng.integers(0, w, n)
    pick_lo = (rng.random(n) < 0.5) & (lo[0, 0] < 0)
    one[np.arange(n), pos] = np.where(pick_lo, lo[0, pos], hi[0, pos])
    fx = fixed[rng.integers(0, len(fixed), n)]
    for k, v in enumerate((None, np.broadcast_to(hi, (n, w)), np.broadcast_to(lo, (n, w)), alt, one, fx)):
        if v is not None:
            out = np.where((mode == k)[:, None], v, out)
    return out


def fe64_rows(rng, mode, bound):
    """Balanced FP64 limbs |limb| <= bound."""
    return _by_mode(rng, mode, [-bound] * 5, [bound] * 5, FIXED51)


def fe_rows(rng, mode):
    """32-bit limbs of fe.cuh up to the largest values fe_carry64 leaves."""
    return _by_mode(rng, mode, [0] * 10, FE_MAX, FIXED25)


def word_rows(rng, mode):
    """32-byte words of values up to 2^255 - 1 (limbs of fe64_frombytes_words up to 2^51 - 1), as eight words."""
    l = _by_mode(rng, mode, [0] * 5, [(1 << 51) - 1] * 5, FIXEDU51)
    return words_of(vals51(l))


def words_of(values):
    return np.array([[(v >> (32 * j)) & 0xffffffff for j in range(8)] for v in values], dtype=np.int64)


def point_rows(rng, n):
    """(n, 20) balanced limbs of four coordinates of scale 1: even items within 2^50 + 2^10 (fe64_finish), odd items
    within 2^50 + 2^14 (the 20-lane carry)."""
    m = modes(rng, n, 4)
    odd = (np.arange(n) % 2 == 1)[:, None]
    return np.concatenate([np.where(odd, fe64_rows(rng, m[:, k], B14), fe64_rows(rng, m[:, k], B10)) for k in range(4)],
                          axis=1)


# ---- the reference formulas, mod p -------------------------------------------------------------------------------------
def to_extended(Xc, Yc, Zc, Tc):                      # curve_models.rs:365-372
    return Xc * Tc % P, Yc * Zc % P, Zc * Tc % P, Xc * Yc % P


def double(X, Y, Z):                                   # curve_models.rs:381-397, then :365-372
    XX, YY, ZZ2 = X * X, Y * Y, 2 * Z * Z
    XpY2 = (X + Y) * (X + Y)
    return to_extended(XpY2 - (YY + XX), YY + XX, YY - XX, ZZ2 - (YY - XX))


def add_pniels(p, q, neg):                             # curve_models.rs:411-452, then :365-372
    X, Y, Z, T = p
    YpX, YmX, Zq, T2d = q
    TT2d, ZZ2 = T * T2d, 2 * Z * Zq
    if not neg:
        PP, MM = (Y + X) * YpX, (Y - X) * YmX
        return to_extended(PP - MM, PP + MM, ZZ2 + TT2d, ZZ2 - TT2d)
    PM, MP = (Y + X) * YmX, (Y - X) * YpX
    return to_extended(PM - MP, PM + MP, ZZ2 - TT2d, ZZ2 + TT2d)


def add_aniels(p, q, neg):                             # curve_models.rs:455-494, then :365-372
    X, Y, Z, T = p
    ypx, ymx, xy2d = q
    Txy2d, Z2 = T * xy2d, Z + Z
    if not neg:
        PP, MM = (Y + X) * ypx, (Y - X) * ymx
        return to_extended(PP - MM, PP + MM, Z2 + Txy2d, Z2 - Txy2d)
    PM, MP = (Y + X) * ymx, (Y - X) * ypx
    return to_extended(PM - MP, PM + MP, Z2 - Txy2d, Z2 + Txy2d)


def as_pniels(q):                                      # edwards.rs:528-535
    X, Y, Z, T = q
    return Y + X, Y - X, Z, T * D2


def assert_coords(got, want, what):
    """got: four lists of coordinate values mod p; want: a list of 4-tuples.  Every coordinate separately."""
    for k, name in enumerate("XYZT"):
        bad = [j for j, w in enumerate(want) if got[k][j] != w[k] % P]
        assert not bad, "%s: coordinate %s wrong for %d items, first %d" % (what, name, len(bad), bad[0])


def assert_within(a, bound, what):
    m = int(np.abs(a).max())
    assert m <= bound, "%s: a limb of magnitude %d exceeds %d" % (what, m, bound)


def assert_fe_scale1(a, what):
    """a: (..., 10k) fe limbs: every limb within scale 1 of fe.cuh."""
    lim = np.tile(np.array(FE_LIM), a.shape[-1] // 10)
    assert (a <= lim).all(), what + ": an fe limb above scale 1"


# ---- 20-lane field -----------------------------------------------------------------------------------------------------
def w20_run(dev, op, a, b=None, n=0):
    nw = a.shape[0] // 4
    out = np.zeros((nw, 32), dtype=np.int64)
    a = np.ascontiguousarray(a.reshape(nw, 20))
    b = np.ascontiguousarray(b.reshape(nw, 20)) if b is not None else None
    assert dev.w20_field_check(op, nw, ptr(a), ptr(b), n, ptr(out)) == 0
    assert (out[:, 20:] == out[:, :12]).all(), "lanes 20..31 do not mirror lanes 0..11"
    return out, out[:, :20].reshape(-1, 5)


def scaled(scale):
    return scale * (1 << 50) + (scale << 14)


@pytest.mark.parametrize("sa,sb", [(1, 1), (2, 2), (3, 2), (2, 3), (1, 4), (1, 7), (7, 1)])
def test_w20_mul_at_the_operand_rule_corners(dev, sa, sb):
    """w20_mul: five splits per lane, a transpose-sum over the group by shuffles and ONE parallel round of carries, at
    scale pairs up to 7 (|a_i b_j| just below 2^103) with the 2^14 slack of the 20-lane carry."""
    rng = np.random.default_rng(100 * sa + sb)
    n = 1 << 16
    a = fe64_rows(rng, modes(rng, n, 1)[:, 0], scaled(sa))
    b = fe64_rows(rng, modes(rng, n, 1)[:, 0], scaled(sb))
    assert scaled(sa) * scaled(sb) < 2**103
    _, got = w20_run(dev, W20_MUL, a, b)
    assert_within(got, B15, "w20_mul")
    want = [x * y % P for x, y in zip(vals51(a), vals51(b))]
    assert [v % P for v in vals51(got)] == want


def test_w20_sq_sqn_carry(dev):
    rng = np.random.default_rng(7)
    n = 1 << 16
    for s in (1, 2):                                        # w20_sq = w20_mul(a, a): scale(a)^2 < 8
        a = fe64_rows(rng, modes(rng, n, 1)[:, 0], scaled(s))
        _, got = w20_run(dev, W20_SQ, a)
        assert_within(got, B15, "w20_sq")
        assert [v % P for v in vals51(got)] == [x * x % P for x in vals51(a)]
    a = fe64_rows(rng, modes(rng, 1 << 12, 1)[:, 0], B14)
    for k in (1, 2, 5, 50):
        _, got = w20_run(dev, W20_SQN, a, n=k)
        assert_within(got, B15, "w20_sqn")
        assert [v % P for v in vals51(got)] == [pow(x, 1 << k, P) for x in vals51(a)], k
    # w20_carry at the scales the point code feeds it (x + y: 2, D - c: 3, 2 ZZ - (YY - XX): 4) ends within the bound;
    # larger integer-valued inputs (53 significant bits, up to 2^62) keep their value
    for s in (1, 2, 3, 4):
        a = fe64_rows(rng, modes(rng, n, 1)[:, 0], scaled(s))
        _, got = w20_run(dev, W20_CARRY, a)
        assert_within(got, B15, "w20_carry")
        assert [v % P for v in vals51(got)] == [v % P for v in vals51(a)]
    mant = rng.integers(0, 1 << 53, size=(n, 5), dtype=np.int64)
    a = (mant << rng.integers(0, 10, size=(n, 5), dtype=np.int64)) * np.where(rng.random((n, 5)) < 0.5, -1, 1)
    _, got = w20_run(dev, W20_CARRY, a)
    assert [v % P for v in vals51(got)] == [v % P for v in vals51(a)]


def test_w20_invert(dev):
    """w20_invert (the fixed chain of fe_invert on w20_mul, every group on its own element): z^(p-2), 0 -> 0, for
    operands of scale < 2."""
    rng = np.random.default_rng(11)
    n = 4096
    m = modes(rng, n, 1)[:, 0]
    a = np.concatenate([fe64_rows(rng, m[:n // 2], B14), fe64_rows(rng, m[n // 2:], int(1.99 * (1 << 50)))])
    _, got = w20_run(dev, W20_INVERT, a)
    assert_within(got, B15, "w20_invert")
    assert [v % P for v in vals51(got)] == [pow(x, P - 2, P) for x in vals51(a)]


def _shared_w20_inputs(rng, n):
    a, b = [], []
    for k, (sa, sb) in enumerate([(1, 1), (2, 2), (3, 2), (2, 3), (1, 4), (1, 7), (7, 1), (1, 1)]):
        a.append(fe64_rows(rng, modes(rng, n // 8, 1)[:, 0], scaled(sa)))
        b.append(fe64_rows(rng, modes(rng, n // 8, 1)[:, 0], scaled(sb)))
    return np.ascontiguousarray(np.concatenate(a)), np.ascontiguousarray(np.concatenate(b))


def test_w20_matches_the_emulated_warp_limb_for_limb(dev, w4):
    """The device build of w20_mul, w20_carry and w20_invert against the host build on an emulated warp: every lane's
    limb equal, not only the value -- both floor the split, both round the carry to nearest even, both apply the same
    carry schedule."""
    rng = np.random.default_rng(13)
    w4.h_w20_raw.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]

    def emulated(op, a, b):
        nw = a.shape[0] // 4
        out = np.zeros((nw, 32), dtype=np.int64)
        w4.h_w20_raw(op, nw, ptr(a), ptr(b), ptr(out))
        return out

    a, b = _shared_w20_inputs(rng, 2048)
    dev_out, _ = w20_run(dev, W20_MUL, a, b)
    assert (dev_out == emulated(0, a, b)).all(), "w20_mul"
    c = np.ascontiguousarray(np.concatenate([fe64_rows(rng, modes(rng, 1024, 1)[:, 0], scaled(s)) for s in (1, 2, 3, 4)]))
    c[:64] = np.array([[(2 * k + 1) << 50, -((2 * k + 1) << 50), 3 << 50, -(3 << 50), 1 << 50] for k in range(64)])  # ties
    dev_out, _ = w20_run(dev, W20_CARRY, c)
    assert (dev_out == emulated(1, c, c)).all(), "w20_carry"
    z = np.ascontiguousarray(fe64_rows(rng, modes(rng, 32, 1)[:, 0], B14))
    dev_out, _ = w20_run(dev, W20_INVERT, z)
    assert (dev_out == emulated(2, z, z)).all(), "w20_invert"


# ---- FP64 chains -------------------------------------------------------------------------------------------------------
def chain_run(dev, op, rows):
    n = rows.shape[0]
    inp = np.zeros((n, 32), dtype=np.int64)
    inp[:, :rows.shape[1]] = rows
    out = np.zeros((n, 32), dtype=np.int64)
    assert dev.chain_check(op, n, ptr(inp), ptr(out)) == 0
    return out


def test_fe64_exponentiation_chains(dev):
    """fe64_pow22501 (both outputs), fe_pow_p58_f64, fe_invert_f64 and x25519_invert against Python pow; every fe64
    output within 2^50 + 2^10 and every fe output within scale 1."""
    rng = np.random.default_rng(17)
    n = 4096
    m = modes(rng, n, 1)[:, 0]
    z = np.concatenate([fe64_rows(rng, m[:n // 2], B10), fe64_rows(rng, m[n // 2:], int(1.99 * (1 << 50)))])
    zv = [v % P for v in vals51(z)]
    out = chain_run(dev, CH_POW22501, z)
    assert_within(out[:, :10], B10, "fe64_pow22501")
    assert [v % P for v in vals51(out[:, :5])] == [pow(x, 2**250 - 1, P) for x in zv]
    assert [v % P for v in vals51(out[:, 5:10])] == [pow(x, 11, P) for x in zv]
    out = chain_run(dev, CH_X25519_INVERT, z)
    assert_within(out[:, :5], B10, "x25519_invert")
    assert [v % P for v in vals51(out[:, :5])] == [pow(x, P - 2, P) for x in zv]
    f = fe_rows(rng, m)
    fv = [v % P for v in vals25(f)]
    for op, e in ((CH_POW_P58, (P - 5) // 8), (CH_INVERT_F64, P - 2)):
        out = chain_run(dev, op, f)
        assert_fe_scale1(out[:, :10], "fe exponentiation")
        want = [pow(x, e, P) for x in fv]
        assert [v % P for v in vals25(out[:, :10])] == want, op
        assert [sum(w << (32 * j) for j, w in enumerate(r)) for r in out[:, 10:18].tolist()] == want, op


def test_fe64_frombytes_accepts_every_255_bit_value(dev):
    """fe64_frombytes_words then fe64_carry on 32-byte words: bit 255 ignored, values in [p, 2^255) kept as they are
    (X25519 accepts them), limbs [0, 2^51) as read and within 2^50 + 2^10 after the carry."""
    rng = np.random.default_rng(19)
    n = 1 << 14
    vals = [int.from_bytes(rng.bytes(32), "little") for _ in range(n // 2)]
    vals += [P + int(x) for x in rng.integers(0, 19, n // 4)]                             # [p, 2^255)
    vals += [2**255 + v for v in vals[:n // 8]] + [2**256 - 1 - k for k in range(n // 8 - len(FIXED))] + list(FIXED)
    w = words_of(vals)
    out = chain_run(dev, CH_FROMBYTES, w)
    v255 = [v % 2**255 for v in vals]
    assert out[:, :5].tolist() == [[(v >> (51 * k)) & ((1 << 51) - 1) for k in range(5)] for v in v255]
    assert_within(out[:, 5:10], B10, "fe64_carry")
    assert [v % P for v in vals51(out[:, 5:10])] == [v % P for v in v255]


def test_fe64_cswap_and_cmov_move_raw_bit_patterns(dev):
    """fe64_cswap / fe64_cmov are XOR-mask moves: any 64-bit pattern (NaN, infinities, -0.0, subnormals) comes out bit
    for bit."""
    rng = np.random.default_rng(23)
    n = 1 << 14
    bits = rng.integers(0, 2**64, size=(n, 10), dtype=np.uint64).view(np.int64)
    special = np.array([0x7ff8000000000000, 0x7ff0000000000001, 0x7ff0000000000000, -0x10000000000000,
                        -0x8000000000000000, 1, -1, 0x4330000000000000], dtype=np.int64)
    bits[:n // 4] = special[rng.integers(0, len(special), size=(n // 4, 10))]
    c = (np.arange(n) % 2).astype(np.int64)[:, None]
    rows = np.concatenate([bits, c], axis=1)
    out = chain_run(dev, CH_CSWAP, rows)
    swap = c.astype(bool)
    assert (out[:, :5] == np.where(swap, bits[:, 5:], bits[:, :5])).all()
    assert (out[:, 5:10] == np.where(swap, bits[:, :5], bits[:, 5:])).all()
    out = chain_run(dev, CH_CMOV, rows)
    assert (out[:, :5] == np.where(swap, bits[:, 5:], bits[:, :5])).all()


# ---- single-thread FP64 point formulas (ge64.cuh) --------------------------------------------------------------------
def ge64_run(dev, op, inp):
    n = inp.shape[0]
    out = np.zeros((n, 20), dtype=np.int64)
    assert dev.ge64_check(op, n, ptr(np.ascontiguousarray(inp)), ptr(out)) == 0
    return out


def _records(rng, n, q_kind):
    """n records of 64 slots: p (balanced, scale 1) at 0; q at 20: 'aniels' / 'pniels' words, 'p3' balanced limbs;
    neg at 60 (alternating)."""
    inp = np.zeros((n, 64), dtype=np.int64)
    inp[:, :20] = point_rows(rng, n)
    qm = modes(rng, n, 4)
    if q_kind == "p3":
        inp[:, 20:40] = point_rows(rng, n)
        q = coords51(inp[:, 20:40])
    else:
        nc = 3 if q_kind == "aniels" else 4
        ws = [word_rows(rng, qm[:, k]) for k in range(nc)]
        for k in range(nc):
            inp[:, 20 + 8 * k:28 + 8 * k] = ws[k]
        q = [[sum(x << (32 * j) for j, x in enumerate(r)) % P for r in w.tolist()] for w in ws]
    inp[:, 60] = np.arange(n) % 2
    return inp, coords51(inp[:, :20]), q


@pytest.mark.parametrize("neg", [0, 1])
def test_ge64_madd_and_padd_off_curve(dev, neg):
    """The bucket kernel's mixed additions: accumulator limbs at scale 1 with both slacks, Niels coordinates as 32-byte
    words up to 2^255 - 1 (limbs up to 2^51 - 1), addition and subtraction."""
    rng = np.random.default_rng(29 + neg)
    for op, kind in ((GE_MADD, "aniels"), (GE_PADD, "pniels")):
        inp, p, q = _records(rng, NPT, kind)
        inp[:, 60] = neg
        got = ge64_run(dev, op, inp)
        assert_within(got, B10, "ge64 add")
        f = add_aniels if kind == "aniels" else add_pniels
        want = [f(pp, qq, neg) for pp, qq in zip(zip(*p), zip(*q))]
        assert_coords(coords51(got), want, "%s neg=%d" % (kind, neg))


def test_ge64_dbl_and_add_p3_off_curve(dev):
    rng = np.random.default_rng(31)
    inp, p, q = _records(rng, NPT, "p3")
    for op in (GE_DBL, GE_DBL_NO_T):
        got = ge64_run(dev, op, inp)
        assert_within(got, B10, "ge64_dbl")
        want = [double(X, Y, Z) for X, Y, Z, _ in zip(*p)]
        c = coords51(got)
        if op == GE_DBL_NO_T:                              # the projective result: T is not computed
            c[3] = [w[3] % P for w in want]
        assert_coords(c, want, "ge64_dbl<%s>" % (op == GE_DBL))
    got = ge64_run(dev, GE_ADD_P3, inp)
    assert_within(got, B10, "ge64_add_p3")
    want = [add_pniels(pp, as_pniels(qq), 0) for pp, qq in zip(zip(*p), zip(*q))]
    assert_coords(coords51(got), want, "ge64_add_p3")


# ---- 4-lane integer point code (warp4.cuh) ---------------------------------------------------------------------------
def fe_point_rows(rng, n):
    m = modes(rng, n, 4)
    return np.concatenate([fe_rows(rng, m[:, k]) for k in range(4)], axis=1)


def w4_run(dev, op, pts, nw, arg=0, first=1):
    pts = np.ascontiguousarray(pts.astype(np.uint32))
    out = np.zeros((nw, 32, 40), dtype=np.uint32)
    st = np.zeros((nw, 8, 40), dtype=np.uint32)
    assert dev.w4_check(op, nw, ptr(pts), pts.shape[0], arg, first, ptr(out), ptr(st)) == 0
    return out, st


def test_w4_add_off_curve(dev):
    """w4_add (k_plain_sum, k_heavy_fixup): as_projective_niels of q, then the projective-Niels addition, in two rounds
    of four products spread over the four lanes of a group.  Coordinates at the largest limbs fe_carry64 leaves; every
    lane's copy is compared, and every output limb must be within scale 1."""
    rng = np.random.default_rng(37)
    n = NPT
    pq = fe_point_rows(rng, 2 * n)
    out, st = w4_run(dev, W4_ADD, pq, n)
    assert (out == out[:, :1]).all(), "the lanes of a warp disagree"
    assert (st == out[:, :1]).all(), "w4_store wrote another value than the lanes hold"
    assert_fe_scale1(out[:, 0], "w4_add")
    p, q = coords25(pq[0::2]), coords25(pq[1::2])
    want = [add_pniels(pp, as_pniels(qq), 0) for pp, qq in zip(zip(*p), zip(*q))]
    assert_coords(coords25(out[:, 0]), want, "w4_add")


def test_w4_and_w4f_shfl_down(dev):
    """w4_shfl_down / w4f_shfl_down: lane l gets the point of lane l + d (multiple of 4), its own above the warp."""
    rng = np.random.default_rng(41)
    nw = 256
    pts = fe_point_rows(rng, 8 * nw)
    recs = np.zeros((8 * nw, 64), dtype=np.int64)
    recs[:, :20] = point_rows(rng, 8 * nw)
    for d in (4, 8, 12, 16, 20, 28):
        src = [(l + d) >> 2 if l + d < 32 else l >> 2 for l in range(32)]
        out, _ = w4_run(dev, W4_SHFL, pts, nw, arg=d)
        assert (out == pts.reshape(nw, 8, 40)[:, src]).all(), d
        got = np.zeros((nw, 32, 20), dtype=np.int64)
        assert dev.w4f_check(W4F_SHFL, nw, ptr(recs), 8 * nw, d, ptr(got)) == 0
        assert (got == recs[:, :20].reshape(nw, 8, 20)[:, src]).all(), d


# ---- 4-lane FP64 point code (warp4_f64.cuh) --------------------------------------------------------------------------
def w4f_run(dev, op, inp, arg=0):
    nw = inp.shape[0]
    out = np.zeros((nw, 32, 20), dtype=np.int64)
    assert dev.w4f_check(op, nw, ptr(np.ascontiguousarray(inp)), nw, arg, ptr(out)) == 0
    assert (out == out[:, :1]).all(), "the lanes of a warp disagree"
    return out[:, 0]


def test_w4f_formulas_off_curve(dev):
    """w4f_dbl (with and without T), w4f_add and w4f_padd (neg 0 and 1): each output coordinate of every lane."""
    rng = np.random.default_rng(43)
    inp, p, q = _records(rng, NPT, "p3")
    for want_t in (1, 0):
        got = w4f_run(dev, W4F_DBL, inp, want_t)
        assert_within(got[:, :20 if want_t else 15], B10, "w4f_dbl")
        want = [double(X, Y, Z) for X, Y, Z, _ in zip(*p)]
        c = coords51(got)
        if not want_t:                                      # T is left as it was
            assert (got[:, 15:20] == inp[:, 15:20]).all()
            c[3] = [w[3] % P for w in want]
        assert_coords(c, want, "w4f_dbl want_t=%d" % want_t)
    got = w4f_run(dev, W4F_ADD, inp)
    assert_within(got, B10, "w4f_add")
    assert_coords(coords51(got), [add_pniels(pp, as_pniels(qq), 0) for pp, qq in zip(zip(*p), zip(*q))], "w4f_add")
    inp, p, q = _records(rng, NPT, "pniels")
    got = w4f_run(dev, W4F_PADD, inp)
    assert_within(got, B10, "w4f_padd")
    want = [add_pniels(pp, qq, k % 2) for k, (pp, qq) in enumerate(zip(zip(*p), zip(*q)))]
    assert_coords(coords51(got), want, "w4f_padd")


# ---- 20-lane point code (warp4_f64.cuh) ------------------------------------------------------------------------------
def w20p_run(dev, op, inp=None, raw=None):
    nw = (inp if inp is not None else raw).shape[0]
    out = np.zeros((nw, 32), dtype=np.int64)
    st = np.zeros((nw, 40), dtype=np.uint32)
    raw = np.ascontiguousarray(raw.astype(np.uint32)) if raw is not None else None
    inp = np.ascontiguousarray(inp) if inp is not None else None
    assert dev.w20_point_check(op, nw, ptr(inp), ptr(raw), ptr(out), ptr(st)) == 0
    assert (out[:, 20:] == out[:, :12]).all(), "lanes 20..31 do not mirror lanes 0..11"
    assert_within(out, B15, "20-lane point")
    return out[:, :20], st.astype(np.int64)


def test_w20_dbl_add_load_store_off_curve(dev):
    rng = np.random.default_rng(47)
    inp, p, q = _records(rng, NPT, "p3")
    got, _ = w20p_run(dev, W20_DBL, inp)
    assert_coords(coords51(got), [double(X, Y, Z) for X, Y, Z, _ in zip(*p)], "w20_dbl")
    got, _ = w20p_run(dev, W20_ADD, inp)
    assert_coords(coords51(got), [add_pniels(pp, as_pniels(qq), 0) for pp, qq in zip(zip(*p), zip(*q))], "w20_add")
    raw = fe_point_rows(rng, NPT)
    got, st = w20p_run(dev, W20_LOAD_STORE, raw=raw)
    assert_within(got, B14, "w20_load")
    want = [tuple(c) for c in zip(*coords25(raw))]
    assert_coords(coords51(got), want, "w20_load")
    assert_fe_scale1(st, "w20_store")
    assert_coords(coords25(st), want, "w20_store")


# ---- on the curve, end to end against the C oracle ---------------------------------------------------------------------
def raw_of(oracle, pts, rnd):
    """Raw fe-limb points (160 bytes each), each multiplied through by a random lambda, so that Z != 1."""
    rows = []
    for Pt in pts:
        l = oracle.p3_limbs(Pt)
        lam = rnd.randrange(1, P)
        for k in range(4):
            v = sum(l[5 * k + i] << (51 * i) for i in range(5)) * lam % P
            rows.append([(v >> s) & m for s, m in zip(SH25, M25)])
    return np.array(rows, dtype=np.int64).reshape(len(pts), 40)


def specials(oracle):
    return [oracle.identity(),
            oracle.decompress((P - 1).to_bytes(32, "little")),          # (0, -1), order 2
            oracle.decompress((0).to_bytes(32, "little"))]              # order 4


def same_point(coords, want_limbs):
    """coords: X, Y, Z, T values; want_limbs: the oracle's 20 limbs.  Equal as projective points, Z != 0."""
    X, Y, Z, T = coords
    Xw, Yw, Zw, Tw = (sum(want_limbs[5 * k + i] << (51 * i) for i in range(5)) for k in range(4))
    return Z % P != 0 and all((a * Zw - b * Z) % P == 0 for a, b in ((X, Xw), (Y, Yw), (T, Tw)))


def combine_cases():
    cases = [(1, 17, 16, 0), (3, 4, 20, 0), (8, 5, 4, 0), (2, 1, 7, 0)]                 # the emulated warp's cases
    ranks = (1, 2, 3, 5, 8, 13, 21, 32)
    for c in range(4, 21):
        r = ranks[c % len(ranks)]
        cases.append((r, max(2, min(math.ceil(256 / c) + 1, 640 // r)), c, c % 3))
    cases.append((32, 3, 5, 1))
    return cases


@pytest.mark.parametrize("ranks,nwin,c,lead", combine_cases())
def test_combine_body_matches_oracle(dev, oracle, ranks, nwin, c, lead):
    """k_combine's body on one warp: w20_horner + w20_encode and w4f_horner give sum_w 2^(c w) sum_r W[r][w]; `lead`
    top windows are empty in every rank; the identity, 2-torsion and 4-torsion points sit first, in the middle and
    last."""
    rnd = random.Random(1000 * ranks + 10 * nwin + c)
    B = oracle.basepoint()
    pts = [oracle.scalarmul(rnd.randrange(pyref.L).to_bytes(32, "little"), B) for _ in range(ranks * nwin)]
    sp = specials(oracle)
    for k, pos in enumerate((0, len(pts) // 2, len(pts) - 1)):
        pts[pos] = sp[(k + c) % 3]
    for r in range(ranks):
        for w in range(nwin - lead, nwin):
            pts[r * nwin + w] = oracle.identity()
    _check_combine(dev, oracle, pts, ranks, nwin, c, rnd)


def test_combine_body_all_identity(dev, oracle):
    rnd = random.Random(5)
    for ranks, nwin, c in ((1, 3, 5), (4, 2, 16), (32, 1, 20)):
        _check_combine(dev, oracle, [oracle.identity()] * (ranks * nwin), ranks, nwin, c, rnd)


def _check_combine(dev, oracle, pts, ranks, nwin, c, rnd):
    want = oracle.identity()
    for w in range(nwin - 1, -1, -1):
        want = oracle.mul_by_pow_2(want, c) if w != nwin - 1 else want
        for r in range(ranks):
            want = oracle.add(want, pts[r * nwin + w])
    raw = np.ascontiguousarray(raw_of(oracle, pts, rnd).astype(np.uint32))
    s = np.zeros((32, 8), dtype=np.uint32)
    pp = np.zeros((32, 40), dtype=np.uint32)
    tot = np.zeros((32, 20), dtype=np.int64)
    assert dev.combine_check(ptr(raw), ranks, nwin, c, ptr(s), ptr(pp), ptr(tot)) == 0
    assert (s == s[:1]).all() and (pp == pp[:1]).all() and (tot == tot[:1]).all(), "the lanes of the warp disagree"
    assert bytes(s[0].tobytes()) == oracle.compress(want)
    pp = pp.astype(np.int64)
    assert_fe_scale1(pp[:1], "w20_encode point")
    assert_within(tot, B15, "w4f_horner")
    wl = oracle.p3_limbs(want)
    P3 = [x[0] for x in coords25(pp[:1])]
    assert same_point(P3, wl)
    assert [x[0] for x in coords51(tot[:1])] == P3             # the replicated total is the very same representation


@pytest.mark.parametrize("kk", [0, 1, 7, 8, 9, 16, 33])
def test_heavy_fixup_tree_matches_oracle(dev, oracle, kk):
    """The body of k_heavy_fixup: eight groups take strided task sums (identity-padded), then the 3-level
    w4_shfl_down / w4_add tree across groups; the old sum of the bucket is folded in by group 0 (first = 0)."""
    rnd = random.Random(kk)
    B = oracle.basepoint()
    nw = 4
    sp = specials(oracle)
    for first in (1, 0):
        pts = [oracle.scalarmul(rnd.randrange(pyref.L).to_bytes(32, "little"), B) for _ in range(nw * (kk + 1))]
        for w in range(nw):
            block = pts[w * (kk + 1):(w + 1) * (kk + 1)]
            for k, pos in enumerate((0, len(block) // 2, len(block) - 1)):
                block[pos] = sp[(k + w) % 3]
            pts[w * (kk + 1):(w + 1) * (kk + 1)] = block
        raw = raw_of(oracle, pts, rnd)
        out, st = w4_run(dev, W4_FIXUP, raw, nw, arg=kk, first=first)
        assert_fe_scale1(out[:, :4], "w4_add tree")
        for w in range(nw):
            block = pts[w * (kk + 1):(w + 1) * (kk + 1)]
            want = oracle.identity() if first else block[0]
            for x in block[1:]:
                want = oracle.add(want, x)
            assert (out[w, :4] == st[w, 0]).all()
            got = [x[0] for x in coords25(st[w, :1])]
            assert same_point(got, oracle.p3_limbs(want)), (kk, first, w)
