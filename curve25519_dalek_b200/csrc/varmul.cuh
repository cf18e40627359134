// varmul.cuh -- constant-time variable-base scalar multiplication s P on the FP64 field (fe64.cuh), host-compilable.
//
// The reference's EdwardsPoint * Scalar (C/backend/serial/scalar_mul/variable_base.rs:11-48):
//   * a LookupTable of [P, 2P, ..., 8P] as projective Niels points (window.rs:97-105);
//   * the radix-16 signed digits of s (scalar.rs:1019-1051; s < 2^255, so the top digit stays in [-8, 8]);
//   * from the top digit down: four doublings (the first three without T, like the reference's projective doublings),
//     then the table entry |d| chosen by a scan of all 8 entries with arithmetic masks and added or subtracted by the
//     masked sign (window.rs:54-76): 63 x 4 doublings, 64 additions.
// Constant time in s: the digits are peeled off shifted registers (no register array is indexed by a digit), every
// table lookup reads all 8 entries at addresses set by the loop counter alone, and the sign is a masked swap inside
// ge64_padd.  The table's storage is the caller's choice (Tab::at(k), k < 8 * VARMUL_ENTRY).
//
// Scale bookkeeping (fe64.cuh:20-22): accumulator coordinates have scale 1; table entries hold Y+X and Y-X at scale 2
// and Z, 2dT at scale 1, so every product of ge64_padd stays below scale 8.
#pragma once
#include "ge64.cuh"
#include "x25519.cuh"

#define VARMUL_ENTRY 20        // doubles per projective Niels entry: YpX | YmX | Z | T2d

// the table in per-thread (local) memory
struct VarmulLocalTab {
    double t[8 * VARMUL_ENTRY];
    FE_HD double &at(int k) { return t[k]; }
};

// EdwardsPoint::as_projective_niels (C/edwards.rs:528-535); d2 = 2d
FE_HD void varmul_to_pniels(ge64_pniels &n, const ge64_p3 &p, const fe64 &d2)
{
    fe64_add(n.YpX, p.Y, p.X);                          // 2
    fe64_sub(n.YmX, p.Y, p.X);                          // 2
    n.Z = p.Z;
    fe64_mul(n.T2d, p.T, d2);
}

template <class Tab>
FE_HD void varmul_store(Tab &tab, int j, const ge64_pniels &e)
{
#pragma unroll
    for (int k = 0; k < 5; k++) {
        tab.at(VARMUL_ENTRY * j + k) = e.YpX.v[k];
        tab.at(VARMUL_ENTRY * j + 5 + k) = e.YmX.v[k];
        tab.at(VARMUL_ENTRY * j + 10 + k) = e.Z.v[k];
        tab.at(VARMUL_ENTRY * j + 15 + k) = e.T2d.v[k];
    }
}

// LookupTable::from (window.rs:97-105): entry j = (j+1) P.  P: scale 1
template <class Tab>
FE_HD void varmul_table(Tab &tab, const ge64_p3 &P)
{
    fe64 d2;
    { fe k; fe_const_2d(k); fe64_from_fe(d2, k); }
    ge64_pniels p1;
    varmul_to_pniels(p1, P, d2);
    varmul_store(tab, 0, p1);
    ge64_p3 acc = P;
#if FE64_DEV
#pragma unroll 1
#endif
    for (int j = 1; j < 8; j++) {
        ge64_padd(acc, acc, p1, 0u);                    // (j+1) P = j P + P
        ge64_pniels e;
        varmul_to_pniels(e, acc, d2);
        varmul_store(tab, j, e);
    }
}

// LookupTable::select (window.rs:54-76) of |d| = xabs in [0, 8]: a masked OR over all 8 entries; 0 gives the identity
// (1, 1, 1, 0).  The sign is applied by the caller's ge64_padd.
template <class Tab>
FE_HD void varmul_select(ge64_pniels &q, Tab &tab, uint32_t xabs)
{
    long long w[VARMUL_ENTRY];
#pragma unroll
    for (int k = 0; k < VARMUL_ENTRY; k++) w[k] = 0;
#if FE64_DEV
#pragma unroll 1
#endif
    for (uint32_t j = 1; j <= 8; j++) {
        const long long m = 0LL - (long long)(xabs == j);
#pragma unroll
        for (int k = 0; k < VARMUL_ENTRY; k++) w[k] |= fe64_bits(tab.at((int)(j - 1) * VARMUL_ENTRY + k)) & m;
    }
    const long long one = fe64_bits(1.0) & (0LL - (long long)(xabs == 0));
    w[0] |= one; w[5] |= one; w[10] |= one;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        q.YpX.v[k] = fe64_from_bits(w[k]); q.YmX.v[k] = fe64_from_bits(w[5 + k]);
        q.Z.v[k] = fe64_from_bits(w[10 + k]); q.T2d.v[k] = fe64_from_bits(w[15 + k]);
    }
}

// Q = s P for s < 2^255 (eight little-endian words; the caller clamps or checks bit 255), P at scale 1.
template <class Tab>
FE_HD void varmul(ge64_p3 &Q, const uint32_t s_in[8], const ge64_p3 &P, Tab &tab)
{
    varmul_table(tab, P);
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = s_in[k];
    // carries of the radix-16 recoding (scalar.rs:1040-1046): bit i of (c1:c0) is the carry into digit i
    uint32_t c0 = 0, c1 = 0, carry = 0;
#pragma unroll
    for (int i = 0; i < 63; i++) {
        const uint32_t nib = (s[i >> 3] >> (4 * (i & 7))) & 15;
        carry = (nib + carry + 8) >> 4;
        if (i + 1 < 32) c0 |= carry << (i + 1); else c1 |= carry << (i + 1 - 32);
    }
    ge64_identity(Q);
    uint32_t cout = 0;                                  // carry out of digit i = carry into digit i + 1
#if FE64_DEV
#pragma unroll 1
#endif
    for (int i = 63; i >= 0; i--) {
        const uint32_t nib = s[7] >> 28;                // digit i = nib + carry in - 16 carry out
#pragma unroll
        for (int k = 7; k > 0; k--) s[k] = (s[k] << 4) | (s[k - 1] >> 28);
        s[0] <<= 4;
        const uint32_t cin = c1 >> 31;
        c1 = (c1 << 1) | (c0 >> 31);
        c0 <<= 1;
        const int d = (int)(nib + cin) - (int)(cout << 4);
        cout = cin;
        if (i < 63) {                                   // the loop counter, not the scalar
            ge64_dbl<false>(Q, Q); ge64_dbl<false>(Q, Q); ge64_dbl<false>(Q, Q); ge64_dbl(Q, Q);
        }
        const int m = d >> 31;
        ge64_pniels q;
        varmul_select(q, tab, (uint32_t)((d + m) ^ m));
        ge64_padd(Q, Q, q, (uint32_t)m & 1u);
    }
}

// BASEPOINT_ORDER l = 2^252 + 27742317777372353535851937790883648493 (C/constants.rs) as eight little-endian words
FE_HD void varmul_order_words(uint32_t l[8])
{
    l[0] = 0x5cf5d3edu; l[1] = 0x5812631au; l[2] = 0xa2f79cd6u; l[3] = 0x14def9deu;
    l[4] = 0; l[5] = 0; l[6] = 0; l[7] = 0x10000000u;
}

FE_HD uint32_t ge64_is_identity(const ge64_p3 &p)
{
    ge_p3 q;
    ge64_to_p3(q, p);
    return ge_is_identity(q);
}

// is_small_order | is_torsion_free << 1 (C/edwards.rs:1405-1437) of P (scale 1): [8]P and [l]P against the identity.
// Points are public: variable time would be allowed, but the same constant-time multiplication serves.
template <class Tab>
FE_HD uint32_t varmul_torsion_flags(const ge64_p3 &P, Tab &tab)
{
    ge64_p3 E;
    ge64_dbl<false>(E, P); ge64_dbl<false>(E, E); ge64_dbl(E, E);
    uint32_t l[8];
    varmul_order_words(l);
    ge64_p3 Q;
    varmul(Q, l, P, tab);
    return ge64_is_identity(E) | (ge64_is_identity(Q) << 1);
}
