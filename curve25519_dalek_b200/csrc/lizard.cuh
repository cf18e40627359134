// lizard.cuh -- Lizard, the injective map from 16-byte strings into ristretto255, and the inverse of the Ristretto
// Elligator map behind it, one item per thread, host-compilable (the host build supplies the SHA-256 compression).
//
//   ristretto_map_to_curve    RistrettoPoint::map_to_curve                    C/ristretto/elligator.rs:62-67
//   lizard_encode             RistrettoPoint::lizard_encode::<Sha256>         C/lizard/lizard_ristretto.rs:25-39
//   lizard_decode             RistrettoPoint::lizard_decode::<Sha256>         :43-71
//   ristretto_to_jacobi       to_jacobi_quartic_ristretto                     :117-188
//   jacobi_e_inv_positive     JacobiPoint::e_inv_positive                     C/lizard/jacobi_quartic.rs:28-63
//   map_to_curve_inverse      RistrettoPoint::map_to_curve_inverse            :78-110, :213-219
//
// The digest is SHA-256 (the reference is generic over a 32-byte Digest and names SHA-256 as the default); every hash
// here is one block: 16 data bytes and the padding.
//
// Constant time: no branch, loop bound or address depends on the payload, the point or a recovered payload.  The
// exceptional cases (X = 0 or Y = 0, s = 0, t = 1, no square root, the tag check, n_found) are masked selects and
// arithmetic; the only loops run a fixed eight times over the Jacobi points, which are picked by masked selects.  The
// inverse square roots run on the FP64 field (fe_sqrt_ratio_i<1>).
//
// Scale bookkeeping (fe.cuh:12-18): every input of a function is scale 1; sums and differences that feed a
// multiplication are carried or noted with their scale.
#pragma once
#include "elligator.cuh"

#if defined(__CUDACC__)
#define LZ_FN __device__ __forceinline__
#else
#define LZ_FN inline
void lizard_host_sha256_compress(uint32_t h[8], uint32_t w[16]);   // supplied by the host build
#endif

LZ_FN void lizard_sha256_compress(uint32_t h[8], uint32_t w[16])
{
#if defined(__CUDACC__)
    sha256_compress_regs(h, w);
#else
    lizard_host_sha256_compress(h, w);
#endif
}

// SHA-256 of 16 bytes (four little-endian words, the bytes in order) -> the 32 digest bytes as eight little-endian words
LZ_FN void lizard_sha256_16(uint32_t dig[8], const uint32_t data[4])
{
    uint32_t h[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 4; k++) w[k] = h2c_bswap32(data[k]);
    w[4] = 0x80000000u;
#pragma unroll
    for (int k = 5; k < 15; k++) w[k] = 0;
    w[15] = 16 * 8;                                  // bit length
    lizard_sha256_compress(h, w);
#pragma unroll
    for (int k = 0; k < 8; k++) dig[k] = h2c_bswap32(h[k]);
}

// The 32 bytes lizard_encode maps (lizard_ristretto.rs:29-36): SHA-256(data) with bytes 8..24 replaced by the data, bit 0
// and the top two bits cleared.  Eight little-endian words.
LZ_FN void lizard_tag(uint32_t out[8], const uint32_t data[4])
{
    uint32_t dig[8];
    lizard_sha256_16(dig, data);
    out[0] = dig[0] & 0xfffffffeu;
    out[1] = dig[1];
#pragma unroll
    for (int k = 0; k < 4; k++) out[2 + k] = data[k];
    out[6] = dig[6];
    out[7] = dig[7] & 0x3fffffffu;
}

// RistrettoPoint::map_to_curve (C/ristretto/elligator.rs:62-67): 32 bytes (bit 255 ignored) -> CompressedRistretto words
LZ_FN void ristretto_map_to_curve(uint32_t out[8], const uint32_t in[8])
{
    fe r0;
    fe_frombytes_words(r0, in);
    ge_p3 P;
    ristretto_elligator(P, r0);
    ristretto_compress<1>(out, P);
}

// RistrettoPoint::lizard_encode::<Sha256> -> CompressedRistretto words.  map_to_curve_restricted's precondition holds by
// construction (bit 0 and bits 254, 255 are clear), so it is map_to_curve.
LZ_FN void lizard_encode(uint32_t out[8], const uint32_t data[4])
{
    uint32_t t[8];
    lizard_tag(t, data);
    ristretto_map_to_curve(out, t);
}

// to_jacobi_quartic_ristretto (lizard_ristretto.rs:117-188): the four Jacobi points (S[k], T[k]) of the representative
// (X, Y, Z) as given (no normalisation: the order of the candidates depends on it).  Outputs scale 1.
LZ_FN void ristretto_to_jacobi(fe S[4], fe T[4], const ge_p3 &P)
{
    fe x2, y2, y4, z2, z_min_y, z_pl_y, z2_min_y2, t, gamma, den, s_over_x, sp_over_xp, tmp, c, iz, iz_min_x, iz_pl_x;
    fe s_over_y, sp_over_yp, one, sqrtm1;
    fe_1(one); fe_const_sqrtm1(sqrtm1);
    fe_sq(x2, P.X);
    fe_sq(y2, P.Y);
    fe_sq(y4, y2);
    fe_sq(z2, P.Z);
    fe_sub(z_min_y, P.Z, P.Y);                       // 3
    fe_add(z_pl_y, P.Z, P.Y);                        // 2
    fe_sub(z2_min_y2, z2, y2);                       // 3
    fe_mul(t, y4, x2);
    fe_mul(t, t, z2_min_y2);                         // Y^4 X^2 (Z^2 - Y^2)
    (void)fe_sqrt_ratio_i<1>(gamma, one, t);         // gamma = invsqrt(...)
    fe_mul(den, gamma, y2);
    fe_mul(s_over_x, den, z_min_y);
    fe_mul(sp_over_xp, den, z_pl_y);
    fe_mul(S[0], s_over_x, P.X);
    fe_mul(t, sp_over_xp, P.X);
    fe_neg(t, t); fe_carry(S[1], t);                 // s1 = -sp_over_xp X
    fe_const_mdouble_invsqrt_a_minus_d(c);
    fe_mul(tmp, c, P.Z);                             // -2/sqrt(-d-1) Z
    fe_mul(T[0], tmp, s_over_x);
    fe_mul(T[1], tmp, sp_over_xp);
    fe_sub(t, y2, z2);                               // 3   -(Z^2 - Y^2)
    fe_const_minvsqrt_one_plus_d(c);
    fe_mul(t, t, c);
    fe_mul(den, t, gamma);                           // -(Z^2 - Y^2) (-1/sqrt(1+d)) gamma
    fe_mul(iz, sqrtm1, P.Z);
    fe_sub(iz_min_x, iz, P.X);                       // 3
    fe_add(iz_pl_x, iz, P.X);                        // 2
    fe_mul(s_over_y, den, iz_min_x);
    fe_mul(sp_over_yp, den, iz_pl_x);
    fe_mul(S[2], s_over_y, P.Y);
    fe_mul(t, sp_over_yp, P.Y);
    fe_neg(t, t); fe_carry(S[3], t);
    fe_const_mdouble_invsqrt_a_minus_d(c);
    fe_mul(tmp, c, iz);
    fe_mul(T[2], tmp, s_over_y);
    fe_mul(T[3], tmp, sp_over_yp);
    // X = 0 or Y = 0: (0, 1), (1, -2i/sqrt(-d-1)), (-1, -2i/sqrt(-d-1)) with the first repeated (s0 = s1 = 0 here)
    const uint32_t xy0 = (uint32_t)(fe_iszero(P.X) | fe_iszero(P.Y));
    fe_const_midouble_invsqrt_a_minus_d(c);
    fe m1; fe_const_minus_one(m1);
    fe_cmov(T[0], one, xy0);
    fe_cmov(T[1], one, xy0);
    fe_cmov(T[2], c, xy0);
    fe_cmov(T[3], c, xy0);
    fe_cmov(S[2], one, xy0);
    fe_cmov(S[3], m1, xy0);
}

// JacobiPoint::e_inv_positive (jacobi_quartic.rs:28-63): the non-negative x with e(x) = (S, T), returned with 1, or zero
// and 0 when there is none.  S, T scale 1; out scale 1.
LZ_FN uint32_t jacobi_e_inv_positive(fe &out, const fe &S, const fe &T)
{
    fe one, a, a2, s2, s4, t, y, x, c;
    fe_1(one);
    const uint32_t s_is_zero = (uint32_t)fe_iszero(S);
    const uint32_t t_is_one = (uint32_t)fe_eq(T, one);
    fe_0(out);
    fe_const_sqrt_id(c);
    fe_cmov(out, c, t_is_one);                       // s = 0: sqrt(i d) if t = 1, else 0
    fe_add(t, T, one);                               // 2
    fe_const_dp1_over_dm1(c);
    fe_mul(a, t, c);                                 // a = (t + 1)(d + 1)/(d - 1)
    fe_sq(a2, a);
    fe_sq(s2, S);
    fe_sq(s4, s2);
    fe_sub(t, s4, a2);                               // 3
    fe_const_sqrtm1(c);
    fe_mul(t, t, c);                                 // i (s^4 - a^2)
    const uint32_t sq = fe_sqrt_ratio_i<1>(y, one, t);
    const uint32_t defined = s_is_zero | sq;
    const uint32_t done = s_is_zero | (1u - sq);
    fe_cneg(s2, (uint32_t)fe_isnegative(S));         // sign(s) s^2, scale <= 2
    fe_carry(s2, s2);
    fe_add(t, a, s2);                                // 2
    fe_mul(x, t, y);
    fe_cneg(x, (uint32_t)fe_isnegative(x));          // the non-negative root
    fe_carry(x, x);
    fe_cmov(out, x, 1u - done);
    fe_0(t);
    fe_cmov(out, t, 1u - defined);                   // None reads as zero (CtOption::unwrap_or(ZERO))
    return defined;
}

// Jacobi point j of the reference's order (jc0, dual(jc0), jc1, dual(jc1), ...) by masked selects over the four
// (no register array is indexed at run time); the dual is (-S, -T).  Outputs scale 1.
LZ_FN void lizard_jacobi_pick(fe &s, fe &t, const fe S[4], const fe T[4], uint32_t j)
{
    s = S[0]; t = T[0];
#pragma unroll
    for (int q = 1; q < 4; q++) {
        const uint32_t hit = (uint32_t)((j >> 1) == (uint32_t)q);
        fe_cmov(s, S[q], hit);
        fe_cmov(t, T[q], hit);
    }
    fe_cneg(s, j & 1u); fe_carry(s, s);
    fe_cneg(t, j & 1u); fe_carry(t, t);
}

// RistrettoPoint::lizard_decode::<Sha256> (lizard_ristretto.rs:43-71) of the representative P: the payload (four words)
// and the number of candidates whose tag checks.  The payload is all zero unless exactly one passes.
//
// Only the eight non-negative candidates are hashed.  A negated candidate cannot pass: it is either zero, which is the
// non-negative candidate it negates (checked already, and the masked SHA-256 of 16 zero bytes is not zero), or odd,
// while the check clears bit 0 of what it compares.  tests/test_lizard_host.py asserts both facts.
LZ_FN uint32_t lizard_decode(uint32_t data[4], const ge_p3 &P)
{
    fe S[4], T[4];
    ristretto_to_jacobi(S, T, P);
#pragma unroll
    for (int k = 0; k < 4; k++) data[k] = 0;
    uint32_t n_found = 0;
#if defined(__CUDACC__)
#pragma unroll 1
#endif
    for (uint32_t j = 0; j < 8; j++) {
        fe s, t, x;
        lizard_jacobi_pick(s, t, S, T, j);
        const uint32_t defined = jacobi_e_inv_positive(x, s, t);
        uint32_t b[8], want[8];
        fe_tobytes_words(b, x);
        lizard_tag(want, b + 2);                     // the payload is bytes 8..24
        uint32_t diff = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) diff |= b[k] ^ want[k];
        const uint32_t ok = defined & (uint32_t)(diff == 0);
        const uint32_t m = 0u - ok;
#pragma unroll
        for (int k = 0; k < 4; k++) data[k] = (data[k] & ~m) | (b[2 + k] & m);
        n_found += ok;
    }
    const uint32_t keep = 0u - (uint32_t)(n_found == 1);
#pragma unroll
    for (int k = 0; k < 4; k++) data[k] &= keep;
    return n_found;
}

// RistrettoPoint::map_to_curve_inverse (lizard_ristretto.rs:213-219) of the representative P: emit(j, words, defined)
// for the 16 candidates, j and j + 8 together (the candidate and its negation; words all zero when it is None).
// Returns the mask (bit j set iff candidate j is Some).
template <typename Emit>
LZ_FN uint32_t map_to_curve_inverse(const ge_p3 &P, Emit emit)
{
    fe S[4], T[4];
    ristretto_to_jacobi(S, T, P);
    uint32_t mask = 0;
#if defined(__CUDACC__)
#pragma unroll 1
#endif
    for (uint32_t j = 0; j < 8; j++) {
        fe s, t, x, nx;
        lizard_jacobi_pick(s, t, S, T, j);
        const uint32_t defined = jacobi_e_inv_positive(x, s, t);
        uint32_t b[8];
        fe_tobytes_words(b, x);
        emit(j, b, defined);
        fe_neg(nx, x);                               // -0 = 0: a None candidate stays zero
        fe_tobytes_words(b, nx);
        emit(j + 8, b, defined);
        mask |= (defined << j) | (defined << (j + 8));
    }
    return mask;
}
