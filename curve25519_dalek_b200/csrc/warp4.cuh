// warp4.cuh -- point operations spread over groups of four lanes.
//
// The tail of an MSM (bucket reduction tree, window Horner) is a chain of dependent point
// operations: latency-bound, not throughput-bound.  Each point operation consists of two stages of
// four independent field multiplications; a group of four adjacent lanes holds the operands
// replicated, every lane multiplies one of the four pairs (ONE fe_mul instruction stream serves the
// four lanes), and the products are exchanged with warp shuffles.  This is the same 4-way split the
// reference's AVX2/IFMA backends use inside one point operation
// (curve25519-dalek/docs/parallel-formulas.md:51-76, src/backend/vector/avx2/edwards.rs:114-296),
// mapped to SIMT lanes instead of SIMD lanes.  All 32 lanes of a warp must execute these calls
// together (full-mask shuffles): callers keep trip counts uniform per warp.
#pragma once
#include "ge.cuh"

struct w4_point { fe X, Y, Z, T; };     // extended point, replicated in the 4 lanes of a group

__device__ __forceinline__ void fe_sel4(fe &o, const fe &a0, const fe &a1, const fe &a2, const fe &a3, uint32_t role)
{
    // branch-free: the four lanes must stay converged so that one fe_mul serves them all
    const uint32_t m0 = 0u - (uint32_t)(role == 0), m1 = 0u - (uint32_t)(role == 1);
    const uint32_t m2 = 0u - (uint32_t)(role == 2), m3 = 0u - (uint32_t)(role == 3);
#pragma unroll
    for (int i = 0; i < 10; i++) o.v[i] = (a0.v[i] & m0) | (a1.v[i] & m1) | (a2.v[i] & m2) | (a3.v[i] & m3);
}

// value held by lane `i` of this lane's group
__device__ __forceinline__ void fe_gbcast(fe &o, const fe &mine, int i)
{
    const int src = (int)((threadIdx.x & 28u) | (uint32_t)i);
#pragma unroll
    for (int k = 0; k < 10; k++) o.v[k] = __shfl_sync(0xffffffffu, mine.v[k], src);
}

__device__ __forceinline__ void w4_identity(w4_point &p) { fe_0(p.X); fe_1(p.Y); fe_1(p.Z); fe_0(p.T); }

__device__ __forceinline__ void w4_load(w4_point &p, const ge_p3_raw *src)
{
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    ge_p3_raw r;
#pragma unroll
    for (int q = 0; q < 10; q++) { uint4 v = s[q]; r.w[4 * q] = v.x; r.w[4 * q + 1] = v.y; r.w[4 * q + 2] = v.z; r.w[4 * q + 3] = v.w; }
#pragma unroll
    for (int i = 0; i < 10; i++) { p.X.v[i] = r.w[i]; p.Y.v[i] = r.w[10 + i]; p.Z.v[i] = r.w[20 + i]; p.T.v[i] = r.w[30 + i]; }
}

// lane `role` stores its quarter (X, Y, Z or T: 40 bytes each) of the point
__device__ __forceinline__ void w4_store(ge_p3_raw *dst, const w4_point &p, uint32_t role)
{
    fe mine; fe_sel4(mine, p.X, p.Y, p.Z, p.T, role);
    uint32_t *o = dst->w + 10 * role;
#pragma unroll
    for (int i = 0; i < 10; i += 2) *reinterpret_cast<uint2 *>(o + i) = make_uint2(mine.v[i], mine.v[i + 1]);
}

// p <- p + q (both extended, curve25519-dalek/src/edwards.rs:795-800 = :528-535 + curve_models.rs:411-430, :365-372)
__device__ __forceinline__ void w4_add(w4_point &p, const w4_point &q, uint32_t role)
{
    fe d2, qYpX, qYmX, qT2d, A, B, f, g, r, a, b, c, zz, D, E, H, DpC, DmC, t;
    fe_const_2d(d2);
    fe_add(t, q.Y, q.X); fe_carry(qYpX, t);
    fe_sub(t, q.Y, q.X); fe_carry(qYmX, t);
    fe_sub(A, p.Y, p.X); fe_add(B, p.Y, p.X);
    fe_mul(qT2d, q.T, d2);                                    // as_projective_niels (replicated)
    fe_sel4(f, A, B, p.T, p.Z, role);                         // a = A*qYmX, b = B*qYpX, c = T*qT2d, zz = Z*qZ
    fe_sel4(g, qYmX, qYpX, qT2d, q.Z, role);
    fe_mul(r, f, g);
    fe_gbcast(a, r, 0); fe_gbcast(b, r, 1); fe_gbcast(c, r, 2); fe_gbcast(zz, r, 3);
    fe_add(D, zz, zz);
    fe_sub(E, b, a); fe_add(H, b, a); fe_add(DpC, D, c); fe_sub(DmC, D, c);
    fe_sel4(f, DmC, DpC, DmC, E, role);                       // X3 = DmC*E, Y3 = DpC*H, Z3 = DmC*DpC, T3 = E*H
    fe_sel4(g, E, H, DpC, H, role);
    fe_mul(r, f, g);
    fe_gbcast(p.X, r, 0); fe_gbcast(p.Y, r, 1); fe_gbcast(p.Z, r, 2); fe_gbcast(p.T, r, 3);
}

// copy of the point held by the group `delta_lanes` lanes above (delta_lanes multiple of 4)
__device__ __forceinline__ void w4_shfl_down(w4_point &o, const w4_point &p, int delta_lanes)
{
#pragma unroll
    for (int i = 0; i < 10; i++) {
        o.X.v[i] = __shfl_down_sync(0xffffffffu, p.X.v[i], delta_lanes);
        o.Y.v[i] = __shfl_down_sync(0xffffffffu, p.Y.v[i], delta_lanes);
        o.Z.v[i] = __shfl_down_sync(0xffffffffu, p.Z.v[i], delta_lanes);
        o.T.v[i] = __shfl_down_sync(0xffffffffu, p.T.v[i], delta_lanes);
    }
}
