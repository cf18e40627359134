// point_ops.cuh -- per-item group arithmetic of the batched point operations (point_ops.cu), host-compilable; the host
// plan of the segmented sum is in ps_plan.h.
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

#include "ge64.cuh"
#include "ps_plan.h"

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
