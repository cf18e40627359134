// msm_batch.cuh -- device code of the batched independent MSMs (msm_batch.cu), host-compilable: the cut of every MSM
// into chunks, the per-term tables and digits, and the chunk loop of both modes on the FP64 field (ge64.cuh).
//
// A chunk is up to MB_CHUNK consecutive terms of one MSM that share one accumulator and its doublings, as the terms of
// a call share them in the reference (straus.rs:129-138, :181-197):
//   variable time   width-5 NAF (scalar.rs:955-1007), tables [A, 3A, ..., 15A] (window.rs:201-211); per digit position
//                   one doubling, then one addition per non-zero digit of the chunk's terms
//   constant time   radix-16 signed digits (scalar.rs:1019-1051), tables [P, 2P, ..., 8P] (window.rs:97-105); per digit
//                   position four doublings, then for every term a masked scan of all eight entries and one addition
//                   whose sign is a mask (window.rs:54-76).  Trip counts depend on the chunk length alone.
// Both tables are eight ge_pniels_packed (1 KiB per term).
#pragma once
#include "straus_vt.cuh"

#define MB_CHUNK 16            // terms per chunk (measured, DESIGN.md §6)

// ---- the cut into chunks: MSM j of n_j terms owns ceil(n_j / MB_CHUNK) chunks, slots chunk_base[j] .. chunk_base[j+1] ----
FE_HD uint32_t mb_chunks(uint64_t n) { return (uint32_t)((n + MB_CHUNK - 1) / MB_CHUNK); }

// the MSM that owns chunk c: the last j in [0, nseg) with chunk_base[j] <= c (empty MSMs own no chunk and are skipped)
FE_HD uint32_t mb_chunk_owner(const uint32_t *chunk_base, uint32_t nseg, uint32_t c)
{
    uint32_t lo = 0, hi = nseg;                                    // chunk_base[lo] <= c < chunk_base[hi]
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (chunk_base[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

// chunk c of the piece -> its MSM, its first term and its length; offsets are the piece's nseg + 1 term offsets
FE_HD void mb_task(uint32_t &seg, uint64_t &first, uint32_t &len, const uint64_t *offsets, const uint32_t *chunk_base, uint32_t nseg,
                   uint32_t c)
{
    seg = mb_chunk_owner(chunk_base, nseg, c);
    first = offsets[seg] + (uint64_t)(c - chunk_base[seg]) * MB_CHUNK;
    const uint64_t left = offsets[seg + 1] - first;
    len = left < MB_CHUNK ? (uint32_t)left : (uint32_t)MB_CHUNK;
}

// ---- per-term preparation ----
// Scalar::as_radix_16 (scalar.rs:1019-1051) of s < 2^255: 64 digits in [-8, 8), the top one in [-8, 8]
FE_HD void mb_radix16(int8_t d[64], const uint32_t s[8])
{
    int carry = 0;
    for (int i = 0; i < 63; i++) {
        const int v = (int)((s[i >> 3] >> (4 * (i & 7))) & 15) + carry;
        carry = (v + 8) >> 4;
        d[i] = (int8_t)(v - (carry << 4));
    }
    d[63] = (int8_t)((int)(s[7] >> 28) + carry);
}

// LookupTable::from (window.rs:97-105): tab = [P, 2P, ..., 8P] as projective Niels points.  P: scale 1
FE_HD void mb_table8(ge_pniels_packed tab[8], const ge64_p3 &P)
{
    fe64 d2; fe64_const_2d(d2);
    ge64_pniels p1;
    fe64_add(p1.YpX, P.Y, P.X); fe64_sub(p1.YmX, P.Y, P.X); p1.Z = P.Z; fe64_mul(p1.T2d, P.T, d2);
    ge64_p3 acc = P;
    ge64_pack_pniels(tab[0], acc, d2);
#if FE64_DEV
#pragma unroll 1
#endif
    for (int j = 1; j < 8; j++) {
        ge64_padd(acc, acc, p1, 0u);                               // (j+1) P = j P + P
        ge64_pack_pniels(tab[j], acc, d2);
    }
}

// LookupTable::select (window.rs:54-76) of |d| = xabs in [0, 8]: a masked OR over all eight packed entries, read at
// addresses set by the loop counter alone; 0 gives the identity (1, 1, 1, 0).  The caller's ge64_padd applies the sign.
FE_HD void mb_select8(ge64_pniels &q, const ge_pniels_packed *tab, uint32_t xabs)
{
    ge_pniels_packed w;
#pragma unroll
    for (int k = 0; k < 32; k++) w.w[k] = 0;
#if FE64_DEV
#pragma unroll 1
#endif
    for (uint32_t j = 1; j <= 8; j++) {
        const uint32_t m = 0u - (uint32_t)(xabs == j);
#if FE64_DEV
        const uint4 *src = reinterpret_cast<const uint4 *>(tab + (j - 1));
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint4 v = src[k];
            w.w[4 * k] |= v.x & m; w.w[4 * k + 1] |= v.y & m; w.w[4 * k + 2] |= v.z & m; w.w[4 * k + 3] |= v.w & m;
        }
#else
        for (int k = 0; k < 32; k++) w.w[k] |= tab[j - 1].w[k] & m;
#endif
    }
    const uint32_t one = (uint32_t)(xabs == 0);
    w.w[0] |= one; w.w[8] |= one; w.w[16] |= one;
    ge64_pniels_unpack(q, w);
}

FE_HD void mb_load_entry(ge64_pniels &q, const ge_pniels_packed *e)
{
    ge_pniels_packed pk;
#if FE64_DEV
    const uint4 *src = reinterpret_cast<const uint4 *>(e);
#pragma unroll
    for (int k = 0; k < 8; k++) { const uint4 v = src[k]; pk.w[4 * k] = v.x; pk.w[4 * k + 1] = v.y; pk.w[4 * k + 2] = v.z; pk.w[4 * k + 3] = v.w; }
#else
    pk = *e;
#endif
    ge64_pniels_unpack(q, pk);
}

// ---- the chunk loops: Q = sum over the chunk's len <= MB_CHUNK terms of s_t P_t ----
// constant time: digits are 64 bytes per term (mb_radix16), tables 8 entries per term (mb_table8)
FE_HD void mb_chunk_ct(ge64_p3 &Q, const int8_t *digits, const ge_pniels_packed *tables, uint32_t len)
{
    ge64_identity(Q);
#if FE64_DEV
#pragma unroll 1
#endif
    for (int i = 63; i >= 0; i--) {
        if (i < 63) {                                              // the loop counter, not a scalar
            ge64_dbl<false>(Q, Q); ge64_dbl<false>(Q, Q); ge64_dbl<false>(Q, Q); ge64_dbl(Q, Q);
        }
#if FE64_DEV
#pragma unroll 1
#endif
        for (uint32_t t = 0; t < len; t++) {
            const int d = digits[64 * t + i];
            const int m = d >> 31;
            ge64_pniels q;
            mb_select8(q, tables + 8 * t, (uint32_t)((d + m) ^ m));
            ge64_padd(Q, Q, q, (uint32_t)m & 1u);
        }
    }
}

// variable time: digits are NAF_LEN bytes per term (naf5), tables 8 entries per term (straus_table5).  The digits
// are read four positions at a time; at each position the chunk's non-zero digits are walked through a bit mask, so
// that a thread spends an addition only where it has one (threads of a warp wait for the busiest of them).
FE_HD void mb_chunk_vt(ge64_p3 &Q, const int8_t *nafs, const ge_pniels_packed *tables, uint32_t len)
{
    ge64_identity(Q);
    bool started = false;                                          // doubling the identity changes nothing
#if FE64_DEV
#pragma unroll 1
#endif
    for (int ib = NAF_LEN / 4 - 1; ib >= 0; ib--) {
        uint32_t w[MB_CHUNK];
        uint32_t any = 0;
        for (uint32_t t = 0; t < len; t++) {
            w[t] = *reinterpret_cast<const uint32_t *>(nafs + (size_t)NAF_LEN * t + 4 * ib);
            any |= w[t];
        }
        if (!any && !started) continue;
#if FE64_DEV
#pragma unroll 1
#endif
        for (int sub = 3; sub >= 0; sub--) {
            uint32_t mask = 0;
            for (uint32_t t = 0; t < len; t++) mask |= (uint32_t)(((w[t] >> (8 * sub)) & 0xffu) != 0) << t;
            if (started) ge64_dbl(Q, Q);
            started = started || mask != 0;
            while (mask) {
#if FE64_DEV
                const uint32_t t = (uint32_t)__ffs((int)mask) - 1u;
#else
                const uint32_t t = (uint32_t)__builtin_ctz(mask);
#endif
                mask &= mask - 1;
                const int d = (int8_t)(w[t] >> (8 * sub));
                const uint32_t neg = d < 0;
                ge64_pniels q;
                mb_load_entry(q, tables + 8 * t + ((uint32_t)(neg ? -d : d) >> 1));      // window.rs:187-192: entry |d| / 2
                ge64_padd(Q, Q, q, neg);
            }
        }
    }
}
