// double_base.cuh -- variable-time double-base scalar multiplication a P + b B on the FP64 field (fe64.cuh / ge64.cuh),
// B the Ed25519 basepoint; host-compilable.  The value of EdwardsPoint::vartime_double_scalar_mul_basepoint
// (C/edwards.rs:1078-1087 -> C/backend/serial/scalar_mul/vartime_double_base.rs:23-72); used by the Ed25519 verifier
// (single.cu, a = k, P = -A, b = s) and by the double-base batch (double_base.cu).
//
// The reference interleaves a width-5 NAF of a over [P, 3P, .., 15P] with a width-8 NAF of b over odd multiples of B and
// skips zero digits.  Here both scalars are cut into radix-16 signed digits (scalar.rs:1019-1051): 63 x 4 doublings,
// at most 64 mixed additions of (|d|) B from an 8-entry affine-Niels table in shared memory and at most 64 additions of
// (|d|) P from the thread's own 8-entry projective-Niels table in local memory.  On SIMT some lane of a warp almost
// always has a non-zero NAF digit at a given position, so skipping zeros saves nothing, while the fixed radix-16
// schedule keeps the lanes in step.  Same group element, hence the same canonical encoding.  Variable time: the digits
// choose branches and table addresses, so a and b must be public.
#pragma once
#include "ge64.cuh"

// radix-16 signed digits of w < 2^255 (Scalar::as_radix_16, scalar.rs:1019-1051): d[0..62] in [-8, 8), d[63] in [-8, 8]
FE_HD void radix16(int8_t d[64], const uint32_t w[8])
{
    int carry = 0;
#if FE64_DEV
#pragma unroll 1
#endif
    for (int pos = 0; pos < 64; pos++) {
        int v = (int)((w[pos >> 3] >> (4 * (pos & 7))) & 15) + carry;
        if (pos < 63) { carry = (v + 8) >> 4; v -= carry << 4; }
        d[pos] = (int8_t)v;
    }
}

// one entry of B's table for double_base_eval: the packed affine Niels point e ((j+1) B, row 0 of the fixed-base table
// of base.cu) as 15 balanced doubles y+x | y-x | 2dxy
FE_HD void double_base_stage_B(double *dst, const ge_niels_packed &e)
{
    ge64_niels q; ge64_niels_unpack(q, e);
    fe64 c;
    fe64_carry(c, q.ypx);  for (int k = 0; k < 5; k++) dst[k] = c.v[k];
    fe64_carry(c, q.ymx);  for (int k = 0; k < 5; k++) dst[5 + k] = c.v[k];
    fe64_carry(c, q.xy2d); for (int k = 0; k < 5; k++) dst[10 + k] = c.v[k];
}

// the per-thread working storage of double_base_eval (local memory): P's table and the digits of both scalars.  The
// caller declares it, so that it sits in the thread's stack frame after the caller's own arrays.
struct DoubleBaseLocal {
    ge64_pniels T[8];                                   // (j+1) P, j = 0..7
    int8_t db[64], da[64];
};

// acc = a P + b B for a, b < 2^255 (eight little-endian words each).  s_B holds (j+1) B, j = 0..7, at s_B + 15 j
// (double_base_stage_B).
FE_HD void double_base_eval(ge64_p3 &acc, const ge_p3 &P, const uint32_t a[8], const uint32_t b[8], const double *s_B,
                            DoubleBaseLocal &w)
{
    ge64_pniels *T = w.T;
    int8_t *db = w.db, *da = w.da;
    {
        ge_p3 Q;
        ge_pniels pn1, pn; ge_p3_to_pniels(pn1, P);
        Q = P;
#if FE64_DEV
#pragma unroll 1
#endif
        for (int j = 0; j < 8; j++) {
            if (j) ge_padd(Q, Q, pn1, 0);
            ge_p3_to_pniels(pn, Q);
            fe64_from_fe(T[j].YpX, pn.YpX); fe64_from_fe(T[j].YmX, pn.YmX); fe64_from_fe(T[j].Z, pn.Z); fe64_from_fe(T[j].T2d, pn.T2d);
        }
    }
    radix16(db, b);
    radix16(da, a);
    ge64_identity(acc);
#if FE64_DEV
#pragma unroll 1
#endif
    for (int pos = 63; pos >= 0; pos--) {
        if (pos != 63) { ge64_dbl(acc, acc); ge64_dbl(acc, acc); ge64_dbl(acc, acc); ge64_dbl(acc, acc); }
        const int x = db[pos], y = da[pos];
        if (x) {
            const int m = x < 0 ? -x : x;
            ge64_niels q;
            const double *row = s_B + 15 * (m - 1);
#pragma unroll
            for (int k = 0; k < 5; k++) { q.ypx.v[k] = row[k]; q.ymx.v[k] = row[5 + k]; q.xy2d.v[k] = row[10 + k]; }
            ge64_madd(acc, acc, q, (uint32_t)(x < 0));
        }
        if (y) {
            const int m = y < 0 ? -y : y;
            ge64_padd(acc, acc, T[m - 1], (uint32_t)(y < 0));
        }
    }
}
