// point_load.cuh -- one input point of a batch call, in any of the C ABI's point formats, as an extended point on the
// device (varmul.cu, lizard.cu).
#pragma once
#include "../../include/dalek_b200.h"
#include "ge.cuh"

// P_j in format FMT -> extended point; an undecodable encoding gives the identity and 0
template <int FMT>
__device__ __forceinline__ uint32_t varmul_load_point(ge_p3 &p, const uint32_t *__restrict__ pts, size_t j)
{
    if constexpr (FMT == DALEK_POINTS_EXTENDED) {
        const uint64_t *l = (const uint64_t *)pts + 20 * j;
        uint64_t c[5];
        fe *dst[4] = {&p.X, &p.Y, &p.Z, &p.T};
#pragma unroll
        for (int q = 0; q < 4; q++) {
#pragma unroll
            for (int k = 0; k < 5; k++) c[k] = l[5 * q + k];
            fe_from_limbs51(*dst[q], c);
        }
        return 1;
    } else {
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = pts[8 * j + k];
    uint32_t good;
    if (FMT == DALEK_POINTS_RISTRETTO) {
        good = ristretto_decompress<1>(p, s);
    } else {
        good = ge_decompress_affine<1>(p.X, p.Y, s);
        fe_1(p.Z);
        fe_mul(p.T, p.X, p.Y);
    }
    ge_p3 id; ge_p3_identity(id);
    const uint32_t bad = 1u - good;
    fe_cmov(p.X, id.X, bad); fe_cmov(p.Y, id.Y, bad); fe_cmov(p.Z, id.Z, bad); fe_cmov(p.T, id.T, bad);
    return good;
    }
}
