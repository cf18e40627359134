// sc.cuh -- arithmetic modulo the group order l = 2^252 + 27742317777372353535851937790883648493
// on 32-bit words.  Values cross this header as 8 little-endian 32-bit words.  Device code under nvcc; a plain C++
// compiler builds it for the host (tests/host/sc_host_check.cpp, tests/host/scalar_ops_host_check.cpp), with SC_L /
// SC_MU as host constants.
//
// Branch-free in the values: every conditional subtraction or addition of l is a masked select, so that the signer
// (sign.cu) can reduce secrets (r, k a + r) here and the scalar batch calls (scalars.cu) can compute on them.  Loop counts
// and the inversion's exponent are fixed.
//
// The reference uses five 52-bit limbs with Montgomery reduction, R = 2^260
// (curve25519-dalek/src/backend/serial/u64/scalar.rs:60-343).  Only canonical values are
// observable, so the device code uses plain Barrett reduction (HAC 14.42, b = 2^32, k = 8): it is
// used a handful of times per signature and is nowhere near the critical path.
#pragma once
#include <stdint.h>

#include "constants.cuh"   // SC_L[8], SC_MU[9]

#if defined(__CUDACC__)
#define SC_HD __device__ __forceinline__     // SC_L / SC_MU are __constant__ here
#else
#define SC_HD inline
#endif

// out[na+nb] = a[na] * b[nb]
template <int NA, int NB>
SC_HD void mp_mul(uint32_t *out, const uint32_t *a, const uint32_t *b)
{
#pragma unroll
    for (int i = 0; i < NA + NB; i++) out[i] = 0;
#pragma unroll
    for (int i = 0; i < NA; i++) {
        uint64_t carry = 0;
#pragma unroll
        for (int j = 0; j < NB; j++) {
            uint64_t t = (uint64_t)a[i] * b[j] + out[i + j] + carry;
            out[i + j] = (uint32_t)t;
            carry = t >> 32;
        }
        out[i + NB] = (uint32_t)carry;
    }
}

// r = a - b over N words, returns borrow
template <int N>
SC_HD uint32_t mp_sub(uint32_t *r, const uint32_t *a, const uint32_t *b)
{
    uint64_t borrow = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
        uint64_t t = (uint64_t)a[i] - b[i] - borrow;
        r[i] = (uint32_t)t;
        borrow = (t >> 63) & 1;
    }
    return (uint32_t)borrow;
}

// 1 if a >= l (a: 8 words)
SC_HD uint32_t sc_ge_l(const uint32_t *a)
{
    uint32_t t[8], l[8];
#pragma unroll
    for (int i = 0; i < 8; i++) l[i] = SC_L[i];
    return 1u - mp_sub<8>(t, a, l);
}

// Scalar::from_canonical_bytes test (C/scalar.rs:259-263): bit 255 clear and value < l
SC_HD uint32_t sc_is_canonical(const uint32_t *a) { return 1u - sc_ge_l(a); }

// x (16 words, < 2^512) mod l -> r (8 words).  Scalar::from_bytes_mod_order_wide value
// (C/scalar.rs:248-250, u64/scalar.rs:89-116).
SC_HD void sc_reduce512(uint32_t *r, const uint32_t *x)
{
    uint32_t mu[9], l[9], q2[18], r2[18];
#pragma unroll
    for (int i = 0; i < 9; i++) mu[i] = SC_MU[i];
#pragma unroll
    for (int i = 0; i < 8; i++) l[i] = SC_L[i];
    l[8] = 0;
    mp_mul<9, 9>(q2, x + 7, mu);              // q1 = x / b^(k-1) (9 words); q2 = q1 * mu
    const uint32_t *q3 = q2 + 9;              // q3 = q2 / b^(k+1) (9 words)
    mp_mul<9, 9>(r2, q3, l);                  // only the low 9 words matter (mod b^(k+1))
    uint32_t t[9];
    mp_sub<9>(t, x, r2);                      // r1 - r2 mod b^9  (0 <= result < 3l)
#pragma unroll 1
    for (int it = 0; it < 2; it++) {                  // t -= l while t >= l, as a masked select
        uint32_t u[9];
        const uint32_t keep = 0u - mp_sub<9>(u, t, l); // all ones: t < l, keep t
#pragma unroll
        for (int i = 0; i < 9; i++) t[i] = (t[i] & keep) | (u[i] & ~keep);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = t[i];
}

// r = a mod l for a 256-bit a (Scalar::from_bytes_mod_order, C/scalar.rs:235-244)
SC_HD void sc_reduce256(uint32_t *r, const uint32_t *a)
{
    uint32_t x[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { x[i] = a[i]; x[8 + i] = 0; }
    sc_reduce512(r, x);
}

// r = a * b mod l (any 256-bit a, b) -- Mul for Scalar (C/scalar.rs:317-322)
SC_HD void sc_mul(uint32_t *r, const uint32_t *a, const uint32_t *b)
{
    uint32_t p[16];
    mp_mul<8, 8>(p, a, b);
    sc_reduce512(r, p);
}

// r = a + b mod l, inputs < l (C/scalar.rs:334-349)
SC_HD void sc_add(uint32_t *r, const uint32_t *a, const uint32_t *b)
{
    uint32_t s[8], u[8], l[8];
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { uint64_t t = (uint64_t)a[i] + b[i] + carry; s[i] = (uint32_t)t; carry = t >> 32; }
#pragma unroll
    for (int i = 0; i < 8; i++) l[i] = SC_L[i];
    const uint32_t keep = 0u - mp_sub<8>(u, s, l);   // inputs < l < 2^253: no carry out of 256 bits
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = (s[i] & keep) | (u[i] & ~keep);
}

// r = -a mod l for a < l (C/scalar.rs:366-374 after its reduction step)
SC_HD void sc_neg(uint32_t *r, const uint32_t *a)
{
    uint32_t l[8], u[8], nz = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { l[i] = SC_L[i]; nz |= a[i]; }
    mp_sub<8>(u, l, a);
    const uint32_t m = 0u - ((nz | (0u - nz)) >> 31);   // all ones iff a != 0
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = u[i] & m;
}

// r = a - b mod l, inputs < l (C/scalar.rs:353-362): l is added back under a mask when the difference borrows
SC_HD void sc_sub(uint32_t *r, const uint32_t *a, const uint32_t *b)
{
    uint32_t d[8];
    const uint32_t m = 0u - mp_sub<8>(d, a, b);      // all ones: a < b
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { uint64_t t = (uint64_t)d[i] + (SC_L[i] & m) + carry; r[i] = (uint32_t)t; carry = t >> 32; }
}

// r = a / 2 mod l for a < l (Scalar::div_by_2, C/scalar.rs:858-870): l is added under a mask when a is odd, then the
// even sum (< 2^254, no carry out of 256 bits) is shifted right by one bit across the words
SC_HD void sc_div_by_2(uint32_t *r, const uint32_t *a)
{
    const uint32_t m = 0u - (a[0] & 1u);
    uint32_t t[8];
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { uint64_t s = (uint64_t)a[i] + (SC_L[i] & m) + carry; t[i] = (uint32_t)s; carry = s >> 32; }
#pragma unroll
    for (int i = 0; i < 7; i++) r[i] = (t[i] >> 1) | (t[i + 1] << 31);
    r[7] = t[7] >> 1;
}

// a^(l-2) mod l by left-to-right square-and-multiply over the bits of l - 2 (uniform control flow: the exponent is public);
// Scalar::invert's value (C/scalar.rs:739-741), 0 for a = 0
SC_HD void sc_invert(uint32_t r[8], const uint32_t a[8])
{
    uint32_t e[8], acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { e[i] = SC_L[i]; acc[i] = i == 0 ? 1u : 0u; }
    e[0] -= 2;                                            // l is odd and l[0] >= 2: no borrow
#pragma unroll 1
    for (int bit = 252; bit >= 0; bit--) {
        sc_mul(acc, acc, acc);
        if ((e[bit >> 5] >> (bit & 31)) & 1) sc_mul(acc, acc, a);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = acc[i];
}
