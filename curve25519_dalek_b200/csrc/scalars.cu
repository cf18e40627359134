// scalars.cu -- scalar batch helpers (SURVEY 8f rank 4):
//   Scalar::from_bytes_mod_order_wide     curve25519-dalek/src/scalar.rs:248-250   k_scalar_from_wide
//   Scalar::invert_batch / _alloc         curve25519-dalek/src/scalar.rs:779-853   k_scalar_invert_groups, k_scalar_product
// The inversion uses Montgomery's trick like the reference (scalar.rs:806-850): a thread owns SC_K consecutive scalars,
// so one exponentiation by l - 2 (scalar.rs:739-741 value; u64/scalar.rs montgomery_invert) is shared by SC_K scalars;
// the product of all inverses that the reference returns is the product of the per-thread inverses.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "sc.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define SC_K 8

// a^(l-2) mod l by left-to-right square-and-multiply over the bits of l - 2 (uniform control flow: the exponent is public)
__device__ __forceinline__ void sc_invert(uint32_t r[8], const uint32_t a[8])
{
    uint32_t e[8], acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { e[i] = SC_L[i]; acc[i] = i == 0 ? 1u : 0u; }
    e[0] -= 2;                                            // l is odd and l[0] >= 2: no borrow
#pragma unroll 1
    for (int bit = 252; bit >= 0; bit--) {
        sc_mul(acc, acc, acc);
        if ((e[bit >> 5] >> (bit & 31)) & 1) sc_mul(acc, acc, a);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = acc[i];
}

__global__ void k_scalar_from_wide(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[16], r[8];
#pragma unroll
    for (int k = 0; k < 16; k++) x[k] = in[16 * i + k];
    sc_reduce512(r, x);
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * i + k] = r[k];
}

// per thread: inverses of SC_K scalars (reduced mod l first); group_inv[t] = inverse of the group's product;
// *zero_flag set if a scalar is 0 mod l (the reference requires nonzero inputs)
__global__ void __launch_bounds__(128)
k_scalar_invert_groups(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out, uint32_t *__restrict__ group_inv,
                       int *__restrict__ zero_flag)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i0 = t * SC_K;
    if (i0 >= n) return;
    uint32_t v[SC_K][8], scratch[SC_K][8], acc[8], tmp[8];
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = k == 0 ? 1u : 0u;
#pragma unroll
    for (int j = 0; j < SC_K; j++) {
        if (i0 + j < n) {
            uint32_t raw[8];
#pragma unroll
            for (int k = 0; k < 8; k++) raw[k] = in[8 * (i0 + j) + k];
            sc_reduce256(v[j], raw);
            uint32_t nz = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) nz |= v[j][k];
            if (!nz) { atomicOr(zero_flag, 1); v[j][0] = 1; }          // keep the group invertible; the call reports the error
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) v[j][k] = k == 0 ? 1u : 0u;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) scratch[j][k] = acc[k];
        sc_mul(acc, acc, v[j]);
    }
    sc_invert(acc, acc);
#pragma unroll
    for (int k = 0; k < 8; k++) group_inv[8 * t + k] = acc[k];
#pragma unroll
    for (int j = SC_K - 1; j >= 0; j--) {
        sc_mul(tmp, acc, v[j]);
        uint32_t o[8];
        sc_mul(o, acc, scratch[j]);
        if (i0 + j < n) {
#pragma unroll
            for (int k = 0; k < 8; k++) out[8 * (i0 + j) + k] = o[k];
        }
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = tmp[k];
    }
}

// product of `count` scalars (one CTA): strided partial products, then a shared-memory tree
__global__ void __launch_bounds__(256) k_scalar_product(const uint32_t *__restrict__ v, size_t count, uint32_t *__restrict__ out)
{
    __shared__ uint32_t sh[256][8];
    uint32_t acc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = k == 0 ? 1u : 0u;
    for (size_t i = threadIdx.x; i < count; i += blockDim.x) {
        uint32_t x[8];
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] = v[8 * i + k];
        sc_mul(acc, acc, x);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) sh[threadIdx.x][k] = acc[k];
    __syncthreads();
    for (uint32_t d = blockDim.x / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            uint32_t a[8], b[8], r[8];
            for (int k = 0; k < 8; k++) { a[k] = sh[threadIdx.x][k]; b[k] = sh[threadIdx.x + d][k]; }
            sc_mul(r, a, b);
            for (int k = 0; k < 8; k++) sh[threadIdx.x][k] = r[k];
        }
        __syncthreads();
    }
    if (threadIdx.x < 8) out[threadIdx.x] = sh[0][threadIdx.x];
}

extern "C" {

int dalek_b200_scalar_from_wide_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n) * 32))) return rc;
    if (n) {
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, in, n * 64, cudaMemcpyHostToDevice, st));
        k_scalar_from_wide<<<cdiv(n, 256), 256, 0, st>>>((const uint32_t *)ctx->ws[WS_STAGING_IN].p, n, (uint32_t *)ctx->ws[WS_SCALARS].p);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(out, ctx->ws[WS_SCALARS].p, n * 32, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return DALEK_OK;
}

int dalek_b200_scalar_invert_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, uint8_t out_product[32])
{
    if (!ctx || !out_product || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    const size_t groups = (n + SC_K - 1) / SC_K;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n) * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], std::max<size_t>(1, groups) * 32 + 64))) return rc;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    if ((rc = pinned_reserve(ctx, 256))) return rc;
    uint32_t *d_groups = (uint32_t *)ctx->ws[WS_STAGING_MSGS].p, *d_prod = d_groups + 8 * std::max<size_t>(1, groups);
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_FLAGS].p, 0, FLAG_WORDS * sizeof(int), st));
    if (n) {
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, in, n * 32, cudaMemcpyHostToDevice, st));
        k_scalar_invert_groups<<<cdiv(groups, 128), 128, 0, st>>>((const uint32_t *)ctx->ws[WS_STAGING_IN].p, n, (uint32_t *)ctx->ws[WS_SCALARS].p, d_groups,
                                                                  (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS);
        ctx->launches++;
    }
    k_scalar_product<<<1, 256, 0, st>>>(d_groups, groups, d_prod);      // empty input: the empty product, 1
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    int *h_zero = (int *)((char *)ctx->h_pinned + 64);
    if (n) CUDA_TRY(ctx, cudaMemcpyAsync(out, ctx->ws[WS_SCALARS].p, n * 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_prod, 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(h_zero, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    if (*h_zero) { ctx->last_error = "invert_batch: a scalar is zero (scalar.rs:796-799: inputs MUST be nonzero)"; return DALEK_E_INVALID_ARG; }
    memcpy(out_product, ctx->h_pinned, 32);
    return DALEK_OK;
}

}  // extern "C"
