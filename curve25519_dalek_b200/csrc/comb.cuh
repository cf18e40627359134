// comb.cuh -- the pieces of a constant-time fixed-base comb shared by the Ristretto double-base batch (straus.cu),
// the X25519 public keys (x25519.cu) and the Ed25519 signer (sign.cu).
//
// A base P is tabulated as 64 rows of 8 entries, entry j of row i = (j+1) 16^i P as balanced FP64 affine Niels
// (15 doubles: y+x | y-x | 2dxy).  s P is then the sum over the 64 radix-16 signed digits d_i of s
// (scalar.rs:1019-1051) of |d_i| 16^i P with the sign of d_i: 64 mixed additions and no doubling.  Every lookup
// scans all 8 entries of its row at warp-uniform addresses with arithmetic masks (window.rs:54-76), and the sign is
// applied by the masked swap / negate inside ge64_madd.
#pragma once
#include "ge64.cuh"

#define COMB_ENTRY 15          // doubles per affine Niels entry

// entry j of row i of the table of `base`: (j+1) 16^i base
__device__ __forceinline__ void comb_entry(double *__restrict__ dst, const ge_p3 &base, int i, int j)
{
    ge_pniels nb; ge_p3_to_pniels(nb, base);
    ge_p3 P = base;
    for (int k = 0; k < j; k++) ge_padd(P, P, nb, 0);            // (j+1) * base
    if (i) ge_mul_by_pow_2(P, P, 4 * i);                         // * 16^i
    fe zi, x, y;
    fe_invert(zi, P.Z);
    fe_mul(x, P.X, zi); fe_mul(y, P.Y, zi);
    ge_niels n; ge_affine_to_niels(n, x, y);
    fe64 e[3];
    fe64_from_fe(e[0], n.ypx); fe64_from_fe(e[1], n.ymx); fe64_from_fe(e[2], n.xy2d);
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int k = 0; k < 5; k++) dst[5 * c + k] = e[c].v[k];
}

// constant-time: select |digit| * 16^i * base from the 8 entries of one table row (digit 0 -> identity)
__device__ __forceinline__ void comb_select(ge64_niels &q, const double *__restrict__ row, uint32_t xabs)
{
    long long w[COMB_ENTRY];
#pragma unroll
    for (int k = 0; k < COMB_ENTRY; k++) w[k] = 0;
#pragma unroll 1
    for (uint32_t j = 1; j <= 8; j++) {
        const long long m = 0LL - (long long)(xabs == j);
#pragma unroll
        for (int k = 0; k < COMB_ENTRY; k++) w[k] |= __double_as_longlong(row[(j - 1) * COMB_ENTRY + k]) & m;
    }
    const long long one = 0x3ff0000000000000LL & (0LL - (long long)(xabs == 0));      // 1.0 for the identity (1, 1, 0)
    w[0] |= one; w[5] |= one;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        q.ypx.v[k] = __longlong_as_double(w[k]); q.ymx.v[k] = __longlong_as_double(w[5 + k]); q.xy2d.v[k] = __longlong_as_double(w[10 + k]);
    }
}

// acc = s B from the table of B in shared memory (64 rows of 8 entries, COMB_ENTRY doubles each), for a secret s < 2^255
// (clamped scalars, reduced scalars): radix-16 signed digits (scalar.rs:1019-1051; s < 2^255 keeps the last digit in range),
// every row scanned in full and the sign applied by the masked negate of ge64_madd, so no branch or address depends on s.
// nibble(pos) returns bits 4 pos .. 4 pos + 3 of s, for pos = 0..63 in order.
template <class Nibble>
__device__ __forceinline__ void comb_mul_base_nibbles(ge64_p3 &acc, const double *__restrict__ s_tab, Nibble nibble)
{
    ge64_identity(acc);
    int carry = 0;
#pragma unroll 1
    for (int pos = 0; pos < 64; pos++) {
        int d = (int)nibble(pos) + carry;
        if (pos < 63) { carry = (d + 8) >> 4; d -= carry << 4; }
        const int m = d >> 31;
        ge64_niels q;
        comb_select(q, s_tab + (size_t)pos * 8 * COMB_ENTRY, (uint32_t)((d + m) ^ m));
        ge64_madd(acc, acc, q, (uint32_t)(d < 0));
    }
}

// the same for s held in registers (consumed: shifted down by one digit per row with funnel shifts, so that no register
// array is indexed at run time)
__device__ __forceinline__ void comb_mul_base(ge64_p3 &acc, uint32_t s[8], const double *__restrict__ s_tab)
{
    comb_mul_base_nibbles(acc, s_tab, [&](int) {
        const uint32_t v = s[0] & 15;
#pragma unroll
        for (int k = 0; k < 7; k++) s[k] = __funnelshift_r(s[k], s[k + 1], 4);
        s[7] >>= 4;
        return v;
    });
}
