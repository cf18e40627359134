// point_ops.cuh -- per-item group arithmetic of the batched point operations (point_ops.cu), host-compilable, and the
// host plan of the segmented sum.
//   Add / Sub          C/edwards.rs:795-835, C/ristretto.rs:838-880        point_apply (PO_ADD, PO_SUB)
//   Neg                C/edwards.rs:853-876, C/ristretto.rs:894-908        point_apply (PO_NEG)
//   Group::double      C/edwards.rs:786-788 (and the Ristretto impl)       point_apply (PO_DOUBLE)
//   mul_by_cofactor    C/edwards.rs:1365-1367                              point_apply (PO_COFACTOR)
//   ct_eq / eq         C/edwards.rs:501-520, C/ristretto.rs:809-832        edwards_eq, ristretto_eq
// A Ristretto point is handled through its Edwards representative: the group law of the coset is the Edwards law, and
// only equality and encoding see the coset.  Element-wise operations run on the integer field (ge.cuh): one addition
// per item is noise next to the exponentiation that decodes it.  The sum adds on the FP64 field (ge64_add_p3), as the
// partial sums of the batched MSM do.
// Constant time in the points: every function here is straight-line in the coordinates; the operation is public.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "ge64.cuh"

enum { PO_ADD = 0, PO_SUB = 1, PO_NEG = 2, PO_DOUBLE = 3, PO_COFACTOR = 4 };

// -P: (-X, Y, Z, -T) (C/edwards.rs:860-871)
FE_HD void point_neg(ge_p3 &r, const ge_p3 &p)
{
    fe t;
    fe_neg(t, p.X); fe_carry(r.X, t);
    fe_neg(t, p.T); fe_carry(r.T, t);
    r.Y = p.Y; r.Z = p.Z;
}

// r = op(a, b); b is read by PO_ADD and PO_SUB only
FE_HD void point_apply(ge_p3 &r, const ge_p3 &a, const ge_p3 &b, int op)
{
    if (op == PO_ADD || op == PO_SUB) {
        ge_pniels n;
        ge_p3_to_pniels(n, b);
        ge_padd(r, a, n, (uint32_t)(op == PO_SUB));
    } else if (op == PO_NEG) {
        point_neg(r, a);
    } else if (op == PO_DOUBLE) {
        ge_dbl(r, a);
    } else {
        ge_mul_by_pow_2(r, a, 3);
    }
}

// X1 Z2 = X2 Z1 and Y1 Z2 = Y2 Z1 (C/edwards.rs:501-512)
FE_HD uint32_t edwards_eq(const ge_p3 &a, const ge_p3 &b)
{
    fe l, r;
    fe_mul(l, a.X, b.Z); fe_mul(r, b.X, a.Z);
    uint32_t e = (uint32_t)fe_eq(l, r);
    fe_mul(l, a.Y, b.Z); fe_mul(r, b.Y, a.Z);
    return e & (uint32_t)fe_eq(l, r);
}

// X1 Y2 = Y1 X2 or X1 X2 = Y1 Y2 (C/ristretto.rs:815-830): equal up to the 4-torsion of the coset
FE_HD uint32_t ristretto_eq(const ge_p3 &a, const ge_p3 &b)
{
    fe l, r;
    fe_mul(l, a.X, b.Y); fe_mul(r, a.Y, b.X);
    const uint32_t e1 = (uint32_t)fe_eq(l, r);
    fe_mul(l, a.X, b.X); fe_mul(r, a.Y, b.Y);
    return e1 | (uint32_t)fe_eq(l, r);
}

// p = c ? identity : p, branch-free
FE_HD void point_cmov_identity(ge_p3 &p, uint32_t c)
{
    ge_p3 id;
    ge_p3_identity(id);
    fe_cmov(p.X, id.X, c); fe_cmov(p.Y, id.Y, c); fe_cmov(p.Z, id.Z, c); fe_cmov(p.T, id.T, c);
}

FE_HD void ge64_cmov_identity(ge64_p3 &p, uint32_t c)
{
    ge64_p3 id;
    ge64_identity(id);
    fe64_cmov(p.X, id.X, c); fe64_cmov(p.Y, id.Y, c); fe64_cmov(p.Z, id.Z, c); fe64_cmov(p.T, id.T, c);
}

// canonical radix-2^51 limbs X | Y | Z | T (what the EXTENDED format and msm_batch's out_limbs hold)
FE_HD void point_to_limbs(uint64_t l[20], const ge_p3 &p)
{
    fe_to_limbs51(l, p.X); fe_to_limbs51(l + 5, p.Y); fe_to_limbs51(l + 10, p.Z); fe_to_limbs51(l + 15, p.T);
}

// ---- the plan of the segmented sum (host) ----
// A level cuts segments (m + 1 offsets) into chunks of at most `chunk` consecutive items that never cross a segment
// boundary.  The chunks tile the items in order, so chunk c covers items [start[c], start[c+1]); segment j owns
// chunks [base[j], base[j+1]) (none when it is empty).  The next level's segments are the chunks' partial sums:
// its offsets are this level's base.
struct PsLevel {
    std::vector<uint32_t> start;    // nchunks + 1
    std::vector<uint32_t> base;     // m + 1
    uint32_t max_len = 0;           // the longest chunk
    uint32_t max_per_seg = 0;       // the most chunks of one segment
};

template <typename Off>
static inline void ps_plan_level(PsLevel &L, const Off *offsets, size_t m, uint32_t chunk)
{
    L.start.clear(); L.base.clear(); L.max_len = 0; L.max_per_seg = 0;
    L.base.reserve(m + 1);
    for (size_t j = 0; j < m; j++) {
        L.base.push_back((uint32_t)L.start.size());
        const uint64_t lo = (uint64_t)offsets[j], hi = (uint64_t)offsets[j + 1];
        uint32_t k = 0;
        for (uint64_t c = lo; c < hi; c += chunk, k++) {
            L.start.push_back((uint32_t)c);
            L.max_len = std::max(L.max_len, (uint32_t)std::min<uint64_t>(chunk, hi - c));
        }
        L.max_per_seg = std::max(L.max_per_seg, k);
    }
    L.base.push_back((uint32_t)L.start.size());
    L.start.push_back(m ? (uint32_t)offsets[m] : 0u);
}

// Pieces of whole chunks of a level with at most `piece` items each (piece >= chunk): cuts[k] .. cuts[k+1] are the
// chunks of piece k.
static inline void ps_pieces(std::vector<uint32_t> &cuts, const std::vector<uint32_t> &start, uint32_t piece)
{
    cuts.assign(1, 0);
    const uint32_t nchunks = (uint32_t)start.size() - 1;
    for (uint32_t c = 0; c < nchunks; c++)
        if (start[c + 1] - start[cuts.back()] > piece) cuts.push_back(c);
    if (cuts.back() != nchunks) cuts.push_back(nchunks);
}
