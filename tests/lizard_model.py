"""Independent big-integer model of Lizard (an injective map from 16-byte strings into ristretto255) and of the inverse of
the Ristretto Elligator map behind it.  TEST INFRASTRUCTURE.

Restates, in plain Python integers and hashlib.sha256, the algorithm the reference's C/lizard/README.md describes:
  * the four Jacobi-quartic points of a Ristretto point (one per even representative up to sign, from one inverse
    square root), with the X = 0 or Y = 0 case;
  * e^-1 on the Jacobi quartic (the non-negative preimage, with the s = 0 and "no square root" cases);
  * map_to_curve_inverse: the 16 candidates (jc0, dual(jc0), ..., jc3, dual(jc3), then their negations);
  * Lizard encode (tag the 16 payload bytes with their SHA-256, clear bit 0 and the top two bits, then MAP) and decode
    (keep the one positive candidate whose tag checks).
Points are extended (X, Y, Z, T) tuples of integers; the candidate order depends on the representative, so nothing here
normalises.  The constants are derived from their definitions."""
import hashlib

from h2c_model import (INVSQRT_A_MINUS_D, SQRT_M1, d, fe_from_bytes, inv, is_negative, p, ristretto_encode,
                       ristretto_map, sqrt_ratio_m1)

# lizard_constants.rs:25-46, from their definitions
SQRT_ID = sqrt_ratio_m1(SQRT_M1 * d % p, 1)[1]                  # +sqrt(i d)
DP1_OVER_DM1 = (d + 1) * inv(d - 1) % p                          # (d + 1) / (d - 1)
MDOUBLE_INVSQRT_A_MINUS_D = (-2 * INVSQRT_A_MINUS_D) % p         # -2 / sqrt(a - d)
MIDOUBLE_INVSQRT_A_MINUS_D = MDOUBLE_INVSQRT_A_MINUS_D * SQRT_M1 % p
MINVSQRT_ONE_PLUS_D = (-sqrt_ratio_m1(1, d + 1)[1]) % p          # -1 / sqrt(1 + d)
assert sqrt_ratio_m1(SQRT_M1 * d % p, 1)[0] and sqrt_ratio_m1(1, d + 1)[0]

# the limbs C/lizard/u64_constants.rs states, radix 2^51
STATED_LIMBS = {
    "SQRT_ID": [2298852427963285, 3837146560810661, 4413131899466403, 3883177008057528, 2352084440532925],
    "DP1_OVER_DM1": [2159851467815724, 1752228607624431, 1825604053920671, 1212587319275468, 253422448836237],
    "MDOUBLE_INVSQRT_A_MINUS_D": [1693982333959686, 608509411481997, 2235573344831311, 947681270984193, 266558006233600],
    "MIDOUBLE_INVSQRT_A_MINUS_D": [1608655899704280, 1999971613377227, 49908634785720, 1873700692181652, 353702208628067],
    "MINVSQRT_ONE_PLUS_D": [321571956990465, 1251814006996634, 2226845496292387, 189049560751797, 2074948709371214],
}
CONSTANTS = {"SQRT_ID": SQRT_ID, "DP1_OVER_DM1": DP1_OVER_DM1, "MDOUBLE_INVSQRT_A_MINUS_D": MDOUBLE_INVSQRT_A_MINUS_D,
             "MIDOUBLE_INVSQRT_A_MINUS_D": MIDOUBLE_INVSQRT_A_MINUS_D, "MINVSQRT_ONE_PLUS_D": MINVSQRT_ONE_PLUS_D}


def from_limbs51(ls):
    return sum(v << (51 * i) for i, v in enumerate(ls)) % p


for _name, _v in CONSTANTS.items():
    assert from_limbs51(STATED_LIMBS[_name]) == _v, _name


def fe_bytes(x):
    return (x % p).to_bytes(32, "little")


def invsqrt(x):
    """FieldElement::invsqrt: sqrt_ratio_i(1, x)."""
    return sqrt_ratio_m1(1, x)


def to_jacobi_quartic(P):
    """to_jacobi_quartic_ristretto (lizard_ristretto.rs:117-188): four (s, t) for the representative (X, Y, Z, T)."""
    X, Y, Z, _ = (c % p for c in P)
    x2, y2, z2 = X * X % p, Y * Y % p, Z * Z % p
    y4 = y2 * y2 % p
    z2_min_y2 = (z2 - y2) % p
    _, gamma = invsqrt(y4 * x2 % p * z2_min_y2 % p)
    den = gamma * y2 % p
    s_over_x = den * (Z - Y) % p
    sp_over_xp = den * (Z + Y) % p
    s0 = s_over_x * X % p
    s1 = (-sp_over_xp * X) % p
    tmp = MDOUBLE_INVSQRT_A_MINUS_D * Z % p
    t0, t1 = tmp * s_over_x % p, tmp * sp_over_xp % p
    den = (-z2_min_y2) * MINVSQRT_ONE_PLUS_D % p * gamma % p
    iz = SQRT_M1 * Z % p
    s_over_y = den * (iz - X) % p
    sp_over_yp = den * (iz + X) % p
    s2 = s_over_y * Y % p
    s3 = (-sp_over_yp * Y) % p
    tmp = MDOUBLE_INVSQRT_A_MINUS_D * iz % p
    t2, t3 = tmp * s_over_y % p, tmp * sp_over_yp % p
    if X == 0 or Y == 0:
        t0 = t1 = 1
        t2 = t3 = MIDOUBLE_INVSQRT_A_MINUS_D
        s2, s3 = 1, p - 1
    return [(s0, t0), (s1, t1), (s2, t2), (s3, t3)]


def x_or_y_is_zero(P):
    return P[0] % p == 0 or P[1] % p == 0


def e_inv_positive(s, t):
    """JacobiPoint::e_inv_positive (jacobi_quartic.rs:28-63): the non-negative preimage of (s, t) under e, or None."""
    s, t = s % p, t % p
    if s == 0:
        return SQRT_ID if t == 1 else 0
    a = (t + 1) * DP1_OVER_DM1 % p
    s2 = s * s % p
    sq, y = invsqrt((s2 * s2 - a * a) * SQRT_M1 % p)
    if not sq:
        return None
    x = (a + (p - s2 if is_negative(s) else s2)) * y % p
    return (p - x) % p if is_negative(x) else x


def elligator_inverse(P):
    """elligator_ristretto_flavor_inverse (lizard_ristretto.rs:78-110): 16 field elements or None."""
    pos = []
    for s, t in to_jacobi_quartic(P):
        pos.append(e_inv_positive(s, t))
        pos.append(e_inv_positive(-s, -t))
    return pos + [None if x is None else (-x) % p for x in pos]


def map_to_curve_inverse(P):
    """RistrettoPoint::map_to_curve_inverse (:213-219): 16 x (32 bytes or None)."""
    return [None if x is None else fe_bytes(x) for x in elligator_inverse(P)]


def map_to_curve_point(b32):
    """RistrettoPoint::map_to_curve (C/ristretto/elligator.rs:62-67) as an extended point."""
    return ristretto_map(fe_from_bytes(b32))


def map_to_curve(b32):
    return ristretto_encode(map_to_curve_point(b32))


def tag(data):
    """The 32 bytes lizard_encode maps: SHA-256(data) with data in bytes 8..24, bit 0 and the top two bits cleared."""
    assert len(data) == 16
    b = bytearray(hashlib.sha256(data).digest())
    b[8:24] = data
    b[0] &= 0xfe
    b[31] &= 0x3f
    return bytes(b)


def lizard_encode_point(data):
    return map_to_curve_point(tag(data))


def lizard_encode(data):
    """RistrettoPoint::lizard_encode::<Sha256> (:25-39) -> CompressedRistretto."""
    return ristretto_encode(lizard_encode_point(data))


def lizard_decode_detail(P):
    """(payload or None, n_found, slot of the passing candidate or None) of lizard_decode::<Sha256> (:43-71)."""
    result, n_found, slot = bytes(16), 0, None
    for j, x in enumerate(elligator_inverse(P)):
        b = fe_bytes(0 if x is None else x)
        if x is not None and tag(b[8:24]) == b:
            result, n_found, slot = b[8:24], n_found + 1, j
    return (result if n_found == 1 else None), n_found, slot


def lizard_decode(P):
    return lizard_decode_detail(P)[0]


# ---------------------------------------------------------------- points and representatives
def ristretto_decode(b32):
    """RFC 9496 4.3.1 DECODE -> extended point with Z = 1, or None."""
    s = int.from_bytes(b32, "little")
    if s >= p or s & 1:
        return None
    ss = s * s % p
    u1, u2 = (1 - ss) % p, (1 + ss) % p
    u2_sqr = u2 * u2 % p
    v = (-(d * u1 * u1) - u2_sqr) % p
    was_square, invsq = invsqrt(v * u2_sqr % p)
    den_x = invsq * u2 % p
    den_y = invsq * den_x * v % p
    x = 2 * s * den_x % p
    if is_negative(x):
        x = p - x
    y = u1 * den_y % p
    t = x * y % p
    if not was_square or is_negative(t) or y == 0:
        return None
    return (x, y, 1, t)


def coset4(P):
    """The four even representatives P + E[4]: (x, y), (i y, i x)-style rotations as extended points."""
    X, Y, Z, T = P
    i = SQRT_M1
    return [(X, Y, Z, T), (Y * i % p, X * i % p, Z, (p - T) % p), ((p - X) % p, (p - Y) % p, Z, T),
            ((p - Y * i % p) % p, (p - X * i % p) % p, Z, (p - T) % p)]


def scale(P, lam):
    return tuple(c * lam % p for c in P)


def to_limbs51(P):
    """20 u64 radix-2^51 limbs (X | Y | Z | T), canonical: the engine's DALEK_POINTS_EXTENDED layout."""
    out = []
    for c in P:
        c %= p
        out += [(c >> (51 * k)) & ((1 << 51) - 1) for k in range(5)]
    return out


def limbs_bytes(P):
    return b"".join(v.to_bytes(8, "little") for v in to_limbs51(P))


IDENTITY = (0, 1, 1, 0)
