// ge64.cuh -- the two mixed additions of the bucket kernel over the FP64 field (fe64.cuh).
// Same formulas as ge_madd / ge_padd in ge.cuh (curve25519-dalek/src/backend/serial/
// curve_models.rs:411-494 followed by :365-372); scale bookkeeping for balanced doubles:
// accumulator coordinates have scale 1, loaded Niels coordinates are in [0, 2^51) (scale 2).
#pragma once
#include "fe64.cuh"
#include "ge.cuh"

struct ge64_p3 { fe64 X, Y, Z, T; };
struct ge64_niels { fe64 ypx, ymx, xy2d; };
struct ge64_pniels { fe64 YpX, YmX, Z, T2d; };

FE_HD void ge64_identity(ge64_p3 &p) { fe64_0(p.X); fe64_1(p.Y); fe64_1(p.Z); fe64_0(p.T); }

FE_HD void ge64_niels_unpack(ge64_niels &n, const ge_niels_packed &o)
{
    fe64_frombytes_words(n.ypx, o.w); fe64_frombytes_words(n.ymx, o.w + 8); fe64_frombytes_words(n.xy2d, o.w + 16);
}
FE_HD void ge64_pniels_unpack(ge64_pniels &n, const ge_pniels_packed &o)
{
    fe64_frombytes_words(n.YpX, o.w); fe64_frombytes_words(n.YmX, o.w + 8);
    fe64_frombytes_words(n.Z, o.w + 16); fe64_frombytes_words(n.T2d, o.w + 24);
}

// shared second half: given a, b, c (scale 1) and D (scale 2) produce r
FE_HD void ge64_add_tail(ge64_p3 &r, const fe64 &a, const fe64 &b, const fe64 &c, const fe64 &D, uint32_t neg)
{
    fe64 E, H, DpC, DmC, F, G;
    fe64_sub(E, b, a);                     // 2
    fe64_add(H, b, a);                     // 2
    fe64_add(DpC, D, c);                   // 3
    fe64_sub(DmC, D, c);                   // 3
    fe64_carry(DmC, DmC);                  // 1   (3 x 3 would break the operand rule of DmC * DpC)
    F = DmC; fe64_cmov(F, DpC, neg);       // T of the completed point
    G = DpC; fe64_cmov(G, DmC, neg);       // Z of the completed point
    fe64_mul(r.X, F, E);                   // <= 3 x 2
    fe64_mul(r.Y, G, H);                   // <= 3 x 2
    fe64_mul(r.Z, DmC, DpC);               // 1 x 3
    fe64_mul(r.T, E, H);                   // 2 x 2
}

// r = p + q (affine Niels), or p - q when neg = 1.   7M
FE_HD void ge64_madd(ge64_p3 &r, const ge64_p3 &p, const ge64_niels &q, uint32_t neg)
{
    FE64_ASSERT_SCALE(p.X, 1); FE64_ASSERT_SCALE(p.Y, 1); FE64_ASSERT_SCALE(p.Z, 1); FE64_ASSERT_SCALE(p.T, 1);
    fe64 A, B, a, b, c, D;
    fe64 qp = q.ypx, qm = q.ymx;
    { fe64 t = qp; fe64_cmov(qp, qm, neg); fe64_cmov(qm, t, neg); }
    fe64_sub(A, p.Y, p.X);                 // 2
    fe64_add(B, p.Y, p.X);                 // 2
    fe64_mul(a, A, qm);                    // 2 x 2
    fe64_mul(b, B, qp);                    // 2 x 2
    fe64_mul(c, p.T, q.xy2d);              // 1 x 2
    fe64_add(D, p.Z, p.Z);                 // 2
    ge64_add_tail(r, a, b, c, D, neg);
}

// r = p + q (projective Niels), or p - q when neg = 1.   8M
FE_HD void ge64_padd(ge64_p3 &r, const ge64_p3 &p, const ge64_pniels &q, uint32_t neg)
{
    FE64_ASSERT_SCALE(p.X, 1); FE64_ASSERT_SCALE(p.Y, 1); FE64_ASSERT_SCALE(p.Z, 1); FE64_ASSERT_SCALE(p.T, 1);
    fe64 A, B, a, b, c, ZZ, D;
    fe64 qp = q.YpX, qm = q.YmX;
    { fe64 t = qp; fe64_cmov(qp, qm, neg); fe64_cmov(qm, t, neg); }
    fe64_sub(A, p.Y, p.X);
    fe64_add(B, p.Y, p.X);
    fe64_mul(a, A, qm);
    fe64_mul(b, B, qp);
    fe64_mul(c, p.T, q.T2d);
    fe64_mul(ZZ, p.Z, q.Z);
    fe64_add(D, ZZ, ZZ);
    ge64_add_tail(r, a, b, c, D, neg);
}

// r = 2p (curve_models.rs:381-397 followed by :365-372).   4S + 4M, two balanced carries.  T_OUT = false leaves r.T
// unset (4S + 3M, the projective result of :357-363), for a doubling that only another doubling reads.
template <bool T_OUT = true>
FE_HD void ge64_dbl(ge64_p3 &r, const ge64_p3 &p)
{
    FE64_ASSERT_SCALE(p.X, 1); FE64_ASSERT_SCALE(p.Y, 1); FE64_ASSERT_SCALE(p.Z, 1);
    fe64 XX, YY, ZZ, XpY, XpY2, Yp, Ym, E, F;
    fe64_sq(XX, p.X);
    fe64_sq(YY, p.Y);
    fe64_sq(ZZ, p.Z);
    fe64_add(XpY, p.X, p.Y); fe64_carry(XpY, XpY);      // squaring needs scale < 2
    fe64_sq(XpY2, XpY);
    fe64_add(Yp, YY, XX);                               // 2
    fe64_sub(Ym, YY, XX);                               // 2
    fe64_sub(E, XpY2, Yp);                              // 3   (X+Y)^2 - Y^2 - X^2
    fe64_add(F, ZZ, ZZ); fe64_sub(F, F, Ym);            // 4   2Z^2 - (Y^2 - X^2)
    fe64_carry(F, F);                                   // 1
    fe64_mul(r.X, E, F);                                // 3 x 1
    fe64_mul(r.Y, Yp, Ym);                              // 2 x 2
    fe64_mul(r.Z, Ym, F);                               // 2 x 1
    if (T_OUT) fe64_mul(r.T, E, Yp);                    // 3 x 2
}

// r = p + q for two extended points on the FP64 field: q -> projective Niels on the fly (edwards.rs:528-535), 9M;
// d2 = 2d (fe64_const_2d)
FE_HD void ge64_add_p3(ge64_p3 &r, const ge64_p3 &p, const ge64_p3 &q, const fe64 &d2)
{
    ge64_pniels pn;
    fe64_add(pn.YpX, q.Y, q.X);                            // 2
    fe64_sub(pn.YmX, q.Y, q.X);                            // 2
    pn.Z = q.Z;
    fe64_mul(pn.T2d, q.T, d2);
    ge64_padd(r, p, pn, 0u);
}

FE_HD void ge64_from_p3(ge64_p3 &o, const ge_p3 &p)
{
    fe64_from_fe(o.X, p.X); fe64_from_fe(o.Y, p.Y); fe64_from_fe(o.Z, p.Z); fe64_from_fe(o.T, p.T);
}

FE_HD void ge64_to_p3(ge_p3 &o, const ge64_p3 &p)
{
    fe64_to_fe(o.X, p.X); fe64_to_fe(o.Y, p.Y); fe64_to_fe(o.Z, p.Z); fe64_to_fe(o.T, p.T);
}

#if defined(__CUDACC__)
// o = p of the lane d above (every lane of the warp takes part): one step of a warp's shuffle tree
__device__ __forceinline__ void ge64_shfl_down(ge64_p3 &o, const ge64_p3 &p, int d)
{
#pragma unroll
    for (int k = 0; k < 5; k++) {
        o.X.v[k] = __shfl_down_sync(0xffffffffu, p.X.v[k], d); o.Y.v[k] = __shfl_down_sync(0xffffffffu, p.Y.v[k], d);
        o.Z.v[k] = __shfl_down_sync(0xffffffffu, p.Z.v[k], d); o.T.v[k] = __shfl_down_sync(0xffffffffu, p.T.v[k], d);
    }
}
#endif
