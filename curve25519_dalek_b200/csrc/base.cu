// base.cu -- fixed-base multiples of the Ed25519 basepoint for PUBLIC scalars: EdwardsPoint::mul_base
// (curve25519-dalek/src/edwards.rs:918-928), e.g. to synthesise benchmark / test points on the device, and the table of B
// that the verifiers read.  Variable-time table indexing: secrets go through the comb of comb.cuh (sign.cu, x25519.cu).
//
// Table: T[i][j] = (j+1) * 16^i * B as packed affine Niels points, i < 64, j < 8 (48 KiB), so that
// s*B = sum_i digit_i * 16^i * B needs 64 mixed additions and no doublings.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "sc.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

__global__ void __launch_bounds__(64) k_build_base_table(ge_niels_packed *__restrict__ table)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 512) return;
    int i = t >> 3, j = t & 7;
    ge_p3 B, P;
    ge_p3_basepoint(B);
    ge_niels nb; ge_affine_to_niels(nb, B.X, B.Y);
    P = B;
    for (int k = 0; k < j; k++) ge_madd(P, P, nb, 0);           // (j+1) B
    if (i) ge_mul_by_pow_2(P, P, 4 * i);                        // * 16^i
    fe zi, x, y;
    fe_invert(zi, P.Z);
    fe_mul(x, P.X, zi); fe_mul(y, P.Y, zi);
    ge_niels n; ge_affine_to_niels(n, x, y);
    ge_niels_packed pk; ge_niels_pack(pk, n);
    table[t] = pk;
}

__device__ __forceinline__ void mul_base(ge_p3 &acc, const uint32_t s_in[8], const ge_niels_packed *__restrict__ table)
{
    // reduce mod l first (B has order l), which also guarantees the radix-16 recoding fits
    uint32_t s[8];
    sc_reduce256(s, s_in);
    ge_p3_identity(acc);
    int carry = 0;
#pragma unroll 1
    for (int i = 0; i < 64; i++) {
        int d = (int)((s[i >> 3] >> (4 * (i & 7))) & 15) + carry;
        carry = (d + 8) >> 4;
        d -= carry << 4;
        if (d != 0) {
            int a = d < 0 ? -d : d;
            const uint4 *src = reinterpret_cast<const uint4 *>(table + (i * 8 + a - 1));
            ge_niels_packed pk;
#pragma unroll
            for (int q = 0; q < 6; q++) { uint4 v = __ldg(src + q); pk.w[4 * q] = v.x; pk.w[4 * q + 1] = v.y; pk.w[4 * q + 2] = v.z; pk.w[4 * q + 3] = v.w; }
            ge_niels n; ge_niels_unpack(n, pk);
            ge_madd(acc, acc, n, (uint32_t)(d < 0));
        }
    }
}

__global__ void __launch_bounds__(128)
k_mul_base(const uint32_t *__restrict__ scalars, size_t n, const ge_niels_packed *__restrict__ table,
           uint64_t *__restrict__ out_limbs, uint32_t *__restrict__ out_comp)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = scalars[8 * i + k];
    ge_p3 P;
    mul_base(P, s, table);
    if (out_limbs) {
        uint64_t *o = out_limbs + 20 * i;
        fe_to_limbs51(o, P.X); fe_to_limbs51(o + 5, P.Y); fe_to_limbs51(o + 10, P.Z); fe_to_limbs51(o + 15, P.T);
    }
    if (out_comp) {
        uint32_t c[8]; ge_compress(c, P);
#pragma unroll
        for (int k = 0; k < 8; k++) out_comp[8 * i + k] = c[k];
    }
}

int base_table_ensure(dalek_b200_ctx *ctx)
{
    if (ctx->base_table_ready) return 0;
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_BASE_TABLE], 512 * sizeof(ge_niels_packed)))) return rc;
    k_build_base_table<<<8, 64, 0, ctx->stream>>>((ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->base_table_ready = true;
    return 0;
}

extern "C" {

int dalek_b200_edwards_mul_base_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, uint64_t *out_limbs,
                                      uint8_t *out_compressed)
{
    if (!ctx || (n && (!scalars || (!out_limbs && !out_compressed)))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    if ((rc = base_table_ensure(ctx))) return rc;
    if (!n) return 0;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], n * 32))) return rc;
    if (out_limbs && (rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], n * 160))) return rc;
    if (out_compressed && (rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], n * 32))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_SCALARS].p, scalars, n * 32, cudaMemcpyHostToDevice, st));
    k_mul_base<<<cdiv(n, 128), 128, 0, st>>>((const uint32_t *)ctx->ws[WS_SCALARS].p, n, (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p,
                                             out_limbs ? (uint64_t *)ctx->ws[WS_STAGING_IN].p : nullptr,
                                             out_compressed ? (uint32_t *)ctx->ws[WS_STAGING_MSGS].p : nullptr);
    ctx->launches++;
    if (out_limbs) CUDA_TRY(ctx, cudaMemcpyAsync(out_limbs, ctx->ws[WS_STAGING_IN].p, n * 160, cudaMemcpyDeviceToHost, st));
    if (out_compressed) CUDA_TRY(ctx, cudaMemcpyAsync(out_compressed, ctx->ws[WS_STAGING_MSGS].p, n * 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
