// x25519.cuh -- the Montgomery ladder on the FP64 field (fe64.cuh), host-compilable.
//
// mont_ladder<NW> is MontgomeryPoint::mul_bits_be (C/montgomery.rs:176-211) over bits nbits-1..0 of an integer of NW
// little-endian 32-bit words (NW = 8 or 16, so up to 512 bits):
//   * u is read with FieldElement::from_bytes: bit 255 ignored, values in [p, 2^255) accepted as they are, twist
//     points accepted;
//   * x0 = identity, x1 = (u : 1), prev = 0; one Costello-Smith algorithm 8 step per bit, then the final swap on
//     the last bit (bit 0);
//   * as_affine: U * W^(p-2), so W = 0 gives u = 0 (montgomery.rs:409-412); nbits = 0 runs no step and gives u = 0.
// x25519(k, u) of x25519-dalek (x25519.rs:390-392) is MontgomeryPoint::mul_clamped (C/montgomery.rs:150-161): the
// 8-word instance over bits 254..0 of the clamped (clamp_integer, C/scalar.rs:1407-1412), NOT reduced k.  Scalar *
// MontgomeryPoint (montgomery.rs:484-492) is the same instance over the unclamped Scalar (bit 255 clear).
// Constant time: nbits is public and uniform per call; the steps run whatever k and u are, the swaps are XOR masks,
// words of k are picked by masks over all NW words (no address depends on k), and the canonical encoding is
// branch-free.
//
// Scale bookkeeping (fe64.cuh:20-22): ladder coordinates have scale 1 between steps; the sums t0, t1, t9, t10 of
// differential_add_and_double have scale 2 and are carried before they are squared (fe64_sq needs scale < 2).
#pragma once
#include "fe64.cuh"

FE_HD long long fe64_bits(double x)
{
#if FE64_DEV
    return __double_as_longlong(x);
#else
    long long r; memcpy(&r, &x, 8); return r;
#endif
}
FE_HD double fe64_from_bits(long long b)
{
#if FE64_DEV
    return __longlong_as_double(b);
#else
    double r; memcpy(&r, &b, 8); return r;
#endif
}

// (a, b) = c ? (b, a) : (a, b)   (c in {0,1}), XOR-mask swap (ProjectivePoint::conditional_swap)
FE_HD void fe64_cswap(fe64 &a, fe64 &b, uint32_t c)
{
    const long long m = 0LL - (long long)c;
#pragma unroll
    for (int i = 0; i < 5; i++) {
        const long long x = fe64_bits(a.v[i]), y = fe64_bits(b.v[i]);
        const long long t = m & (x ^ y);
        a.v[i] = fe64_from_bits(x ^ t);
        b.v[i] = fe64_from_bits(y ^ t);
    }
}

// clamp_integer (C/scalar.rs:1407-1412) on eight little-endian words
FE_HD void x25519_clamp(uint32_t k[8])
{
    k[0] &= 0xfffffff8u;
    k[7] &= 0x7fffffffu;
    k[7] |= 0x40000000u;
}

// k[w] selected by masks over all NW words: the word index never becomes a register-array address
template <int NW = 8>
FE_HD uint32_t x25519_word(const uint32_t k[NW], int w)
{
    uint32_t r = 0;
#pragma unroll
    for (int j = 0; j < NW; j++) r |= k[j] & (0u - (uint32_t)(j == w));
    return r;
}

// z^(p-2) with the fixed chain of fe_invert_f64 (fe64_pow22501); 0 -> 0.  z: scale < 2; output scale 1
FE_HD void x25519_invert(fe64 &r, const fe64 &z)
{
    fe64 t19, t3;
    fe64_pow22501(t19, t3, z);
    fe64_sqn(t19, t19, 5);
    fe64_mul(r, t19, t3);
}

// canonical little-endian encoding (FieldElement::to_bytes) of f (scale <= 4)
FE_HD void x25519_encode(uint32_t w[8], const fe64 &f)
{
    fe o;
    fe64_to_fe(o, f);
    fe_tobytes_words(w, o);
}

// SharedSecret::was_contributory (x25519.rs:335-337): 1 unless all 32 bytes are zero; branch-free
FE_HD uint32_t x25519_contributory(const uint32_t w[8])
{
    uint32_t d = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) d |= w[j];
    return (d | (0u - d)) >> 31;
}

// differential_add_and_double (C/montgomery.rs:430-468): (U0 : W0) <- 2 P, (U1 : W1) <- P + Q, with u = u(P - Q).
// 6M + 4S per step: t13 = ((A + 2) / 4) * t6 is a full multiplication by the constant 121666.
FE_HD void x25519_ladder_step(fe64 &U0, fe64 &W0, fe64 &U1, fe64 &W1, const fe64 &u)
{
    FE64_ASSERT_SCALE(U0, 1); FE64_ASSERT_SCALE(W0, 1); FE64_ASSERT_SCALE(U1, 1); FE64_ASSERT_SCALE(W1, 1);
    fe64 a24; fe64_0(a24); a24.v[0] = 121666.0;
    fe64 t0, t1, t2, t3, t4, t5, t6, t7, t8, t9, t10, t13, t15;
    fe64_add(t0, U0, W0); fe64_carry(t0, t0);          // 1
    fe64_sub(t1, U0, W0); fe64_carry(t1, t1);          // 1
    fe64_add(t2, U1, W1);                              // 2
    fe64_sub(t3, U1, W1);                              // 2
    fe64_sq(t4, t0);                                   // (U_P + W_P)^2
    fe64_sq(t5, t1);                                   // (U_P - W_P)^2
    fe64_sub(t6, t4, t5);                              // 2   4 U_P W_P
    fe64_mul(t7, t0, t3);                              // 1 x 2
    fe64_mul(t8, t1, t2);                              // 1 x 2
    fe64_add(t9, t7, t8); fe64_carry(t9, t9);          // 1   2 (U_P U_Q - W_P W_Q)
    fe64_sub(t10, t7, t8); fe64_carry(t10, t10);       // 1   2 (W_P U_Q - U_P W_Q)
    fe64_mul(t13, a24, t6);                            // tiny x 2
    fe64_add(t15, t13, t5);                            // 2
    fe64_mul(U0, t4, t5);                              // t14: U of 2P
    fe64_mul(W0, t6, t15);                             // t16: W of 2P   (2 x 2)
    fe64_sq(U1, t9);                                   // t18 = t11: U of P + Q
    fe64_sq(t10, t10);                                 // t12
    fe64_mul(W1, u, t10);                              // t17: W of P + Q
}

// out = u([n] P) for u = u(P) (u_in: eight little-endian words) and n = bits nbits-1..0 of k (NW words, nbits <= 32 NW),
// as eight canonical little-endian words (montgomery.rs:176-211, :409-412)
template <int NW>
FE_HD void mont_ladder(uint32_t out[8], const uint32_t k[NW], int nbits, const uint32_t u_in[8])
{
    fe64 u, U0, W0, U1, W1;
    fe64_frombytes_words(u, u_in);                     // bit 255 ignored, [p, 2^255) accepted (montgomery.rs:598-605)
    fe64_carry(u, u);                                  // scale 1
    fe64_1(U0); fe64_0(W0);                            // x0 = identity
    U1 = u; fe64_1(W1);                                // x1 = (u : 1)
    uint32_t prev = 0;
#if FE64_DEV
#pragma unroll 1
#endif
    for (int i = nbits - 1; i >= 0; i--) {
        const uint32_t bit = (x25519_word<NW>(k, i >> 5) >> (i & 31)) & 1u;
        const uint32_t swap = prev ^ bit;
        fe64_cswap(U0, U1, swap);
        fe64_cswap(W0, W1, swap);
        x25519_ladder_step(U0, W0, U1, W1, u);
        prev = bit;
    }
    fe64_cswap(U0, U1, prev);                          // prev = bit 0 of n (0 when nbits = 0)
    fe64_cswap(W0, W1, prev);
    fe64 wi, r;
    x25519_invert(wi, W0);
    fe64_mul(r, U0, wi);
    x25519_encode(out, r);
}

// out = x25519(k, u) as eight canonical little-endian words (montgomery.rs:150-211, :409-412)
FE_HD void x25519_ladder(uint32_t out[8], const uint32_t k_in[8], const uint32_t u_in[8])
{
    uint32_t k[8];
#pragma unroll
    for (int j = 0; j < 8; j++) k[j] = k_in[j];
    x25519_clamp(k);
    mont_ladder<8>(out, k, 255, u_in);
}
