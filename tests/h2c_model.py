"""Independent big-integer model of hashing into ristretto255 and edwards25519.  TEST INFRASTRUCTURE.

Restates, in plain Python integers and hashlib.sha512:
  * RFC 9496 4.2 SQRT_RATIO_M1, 4.3.2 ENCODE, 4.3.4 MAP and the one-way map (from_uniform_bytes);
  * RFC 9380 5.3.1 expand_message_xmd, 5.2 hash_to_field (m = 1, L = 48), 6.7.1 map_to_curve_elligator2 (the generic
    form, not the straight-line G.2.1 that the engine runs), Appendix D's rational map to edwards25519 with its
    exceptional case, and cofactor clearing (h_eff = 8).
Used to write tests/golden/hash_to_curve.json and to cross-check the engine, the host build and the C oracle."""
import hashlib

p = 2**255 - 19
d = (-121665 * pow(121666, p - 2, p)) % p
SQRT_M1 = pow(2, (p - 1) // 4, p)
J = 486662


def inv(x):
    return pow(x, p - 2, p)


def is_negative(x):
    return (x % p) & 1


def ct_abs(x):
    x %= p
    return (p - x) % p if x & 1 else x


def sqrt_ratio_m1(u, v):
    """RFC 9496 4.2: (was_square, nonnegative r) with r^2 v = u, or r^2 v = SQRT_M1 u when u / v is not a square."""
    u %= p
    v %= p
    r = u * pow(v, 3, p) * pow(u * pow(v, 7, p), (p - 5) // 8, p) % p
    check = v * r * r % p
    correct = check == u
    flipped = check == (-u) % p
    flipped_i = check == (-u * SQRT_M1) % p
    if flipped or flipped_i:
        r = r * SQRT_M1 % p
    return correct or flipped, ct_abs(r)


def _root(square, sign):
    ok, r = sqrt_ratio_m1(square, 1)
    assert ok
    return r if sign == 0 else (p - r) % p


# RFC 9496 4.1 constants, from their definitions
ONE_MINUS_D_SQ = (1 - d * d) % p
D_MINUS_ONE_SQ = (d - 1) ** 2 % p
SQRT_AD_MINUS_ONE = 25063068953384623474111414158702152701244531502492656460079210482610430750235
INVSQRT_A_MINUS_D = 54469307008909316920995813868745141605393597292927456921205312896311721017578
assert SQRT_AD_MINUS_ONE ** 2 % p == (-d - 1) % p
assert INVSQRT_A_MINUS_D ** 2 * (-1 - d) % p == 1
# RFC 9380 G.2.2: c1 = sqrt(-486664) with sgn0(c1) = 0
SQRT_M486664 = _root(-486664, 0)


# ---------------------------------------------------------------- ristretto255 (RFC 9496)
def ext_add(P, Q):
    """Complete addition on -x^2 + y^2 = 1 + d x^2 y^2 in extended coordinates (X : Y : Z : T)."""
    X1, Y1, Z1, T1 = P
    X2, Y2, Z2, T2 = Q
    A = (Y1 - X1) * (Y2 - X2) % p
    B = (Y1 + X1) * (Y2 + X2) % p
    C = T1 * 2 * d * T2 % p
    D = Z1 * 2 * Z2 % p
    E, F, G, H = B - A, D - C, D + C, B + A
    return (E * F % p, G * H % p, F * G % p, E * H % p)


def ristretto_map(t):
    """RFC 9496 4.3.4 MAP on a field element t: an extended point."""
    r = SQRT_M1 * t * t % p
    u = (r + 1) * ONE_MINUS_D_SQ % p
    v = (-1 - r * d) * (r + d) % p
    was_square, s = sqrt_ratio_m1(u, v)
    s_prime = (-ct_abs(s * t)) % p
    s = s if was_square else s_prime
    c = p - 1 if was_square else r
    N = (c * (r - 1) * D_MINUS_ONE_SQ - v) % p
    w0 = 2 * s * v % p
    w1 = N * SQRT_AD_MINUS_ONE % p
    w2 = (1 - s * s) % p
    w3 = (1 + s * s) % p
    return (w0 * w3 % p, w2 * w1 % p, w1 * w3 % p, w0 * w2 % p)


def map_inputs(r0):
    """(N_s, D) of the reference's map for a field element r0: D = 0 makes sqrt_ratio_i(N_s, 0) return (false, 0)."""
    r = SQRT_M1 * r0 * r0 % p
    return (r + 1) * ONE_MINUS_D_SQ % p, (-1 - d * r) * (r + d) % p


def ns_d_is_square(r0):
    ns, dd = map_inputs(r0)
    return sqrt_ratio_m1(ns, dd)[0]


def ristretto_encode(P):
    """RFC 9496 4.3.2 ENCODE."""
    x0, y0, z0, t0 = P
    u1 = (z0 + y0) * (z0 - y0) % p
    u2 = x0 * y0 % p
    _, invsqrt = sqrt_ratio_m1(1, u1 * u2 * u2)
    den1 = invsqrt * u1 % p
    den2 = invsqrt * u2 % p
    z_inv = den1 * den2 * t0 % p
    ix0, iy0 = x0 * SQRT_M1 % p, y0 * SQRT_M1 % p
    enchanted = den1 * INVSQRT_A_MINUS_D % p
    rotate = is_negative(t0 * z_inv)
    x, y = (iy0, ix0) if rotate else (x0, y0)
    den_inv = enchanted if rotate else den2
    if is_negative(x * z_inv):
        y = (-y) % p
    s = ct_abs(den_inv * (z0 - y))
    return s.to_bytes(32, "little")


def fe_from_bytes(b):
    """FieldElement::from_bytes: bit 255 ignored."""
    return (int.from_bytes(b, "little") & ((1 << 255) - 1)) % p


def ristretto_elligator(r0_bytes):
    """compress(MAP(r0)) with r0 read like FieldElement::from_bytes (the elligator_vs_ristretto_sage vectors)."""
    return ristretto_encode(ristretto_map(fe_from_bytes(r0_bytes)))


def from_uniform_bytes(b64):
    """RFC 9496 4.3.4 one-way map: MAP of both halves, then the sum."""
    assert len(b64) == 64
    return ristretto_encode(ext_add(ristretto_map(fe_from_bytes(b64[:32])), ristretto_map(fe_from_bytes(b64[32:]))))


def hash_from_bytes(msg):
    """RistrettoPoint::hash_from_bytes::<Sha512>: the one-way map of SHA-512(msg)."""
    return from_uniform_bytes(hashlib.sha512(msg).digest())


# ---------------------------------------------------------------- RFC 9380, edwards25519_XMD:SHA-512_ELL2
def expand_message_xmd(msg, dst, len_in_bytes):
    """RFC 9380 5.3.1 with H = SHA-512 (b_in_bytes = 64, s_in_bytes = 128)."""
    assert 1 <= len(dst) <= 255
    ell = -(-len_in_bytes // 64)
    assert ell <= 255 and len_in_bytes <= 65535
    dst_prime = dst + bytes([len(dst)])
    msg_prime = bytes(128) + msg + len_in_bytes.to_bytes(2, "big") + b"\0" + dst_prime
    b0 = hashlib.sha512(msg_prime).digest()
    b = [hashlib.sha512(b0 + b"\x01" + dst_prime).digest()]
    for i in range(2, ell + 1):
        b.append(hashlib.sha512(bytes(x ^ y for x, y in zip(b0, b[-1])) + bytes([i]) + dst_prime).digest())
    return b"".join(b)[:len_in_bytes]


def hash_to_field(msg, dst, count):
    """RFC 9380 5.2 with m = 1, L = 48."""
    ub = expand_message_xmd(msg, dst, 48 * count)
    return [int.from_bytes(ub[48 * i:48 * i + 48], "big") % p for i in range(count)]


def from_bytes_wide(b64):
    """FieldElement::from_bytes_wide: the 64 bytes as a little-endian integer, mod p."""
    return int.from_bytes(b64, "little") % p


def is_square(x):
    x %= p
    return x == 0 or pow(x, (p - 1) // 2, p) == 1


def sqrt_with_sign(x, sign):
    ok, r = sqrt_ratio_m1(x, 1)
    assert ok
    return r if sign == 0 else (p - r) % p


def elligator2(u):
    """RFC 9380 6.7.1 map_to_curve_elligator2 for curve25519 (J = 486662, K = 1, Z = 2): Montgomery (s, t)."""
    u %= p
    den = (1 + 2 * u * u) % p
    x1 = (-J) * (inv(den) if den else 0) % p
    if x1 == 0:
        x1 = (-J) % p
    gx1 = (x1 ** 3 + J * x1 * x1 + x1) % p
    x2 = (-x1 - J) % p
    gx2 = (x2 ** 3 + J * x2 * x2 + x2) % p
    if is_square(gx1):
        x, y = x1, sqrt_with_sign(gx1, 1)
    else:
        x, y = x2, sqrt_with_sign(gx2, 0)
    return x, y


def rational_map(s, t):
    """RFC 9380 Appendix D: curve25519 (s, t) -> edwards25519 (v, w); the exceptional points go to the identity."""
    if t % p == 0 or (s + 1) % p == 0:
        return (0, 1)
    return (SQRT_M486664 * s * inv(t) % p, (s - 1) * inv(s + 1) % p)


def exceptional(u):
    s, t = elligator2(u)
    return t % p == 0 or (s + 1) % p == 0


def map_to_curve(u):
    return rational_map(*elligator2(u))


def _aff_add(P, Q):
    x1, y1 = P
    x2, y2 = Q
    k = d * x1 * x2 * y1 * y2 % p
    return ((x1 * y2 + x2 * y1) * inv(1 + k) % p, (y1 * y2 + x1 * x2) * inv(1 - k) % p)


def clear_cofactor(P):
    for _ in range(3):
        P = _aff_add(P, P)
    return P


def compress_edwards(P):
    x, y = P
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


def hash_to_curve(msg, dst):
    """edwards25519_XMD:SHA-512_ELL2_RO_ (RFC 9380 3, 6.8.2): CompressedEdwardsY."""
    u0, u1 = hash_to_field(msg, dst, 2)
    return compress_edwards(clear_cofactor(_aff_add(map_to_curve(u0), map_to_curve(u1))))


def encode_to_curve(msg, dst):
    """edwards25519_XMD:SHA-512_ELL2_NU_: CompressedEdwardsY."""
    (u0,) = hash_to_field(msg, dst, 1)
    return compress_edwards(clear_cofactor(map_to_curve(u0)))


def map_to_curve_compressed(u):
    """compress(map_to_curve(u)) without cofactor clearing (what the host build's map gives)."""
    return compress_edwards(map_to_curve(u))


def d_zero_halves():
    """The four r0 with D = (-1 - d r)(r + d) = 0, r = i r0^2: r0 = +-sqrt(r / i) for r = -d and r = -1/d."""
    out = []
    for r in ((-d) % p, (-inv(d)) % p):
        ok, root = sqrt_ratio_m1(r * inv(SQRT_M1), 1)
        assert ok, "r / i is a square for both roots of D"
        out += [root, (p - root) % p]
    for r0 in out:
        assert map_inputs(r0)[1] == 0
    return out
