// x25519.cu -- X25519 key agreement and public-key derivation in bulk (x25519-dalek, RFC 7748).
//   x25519(k, u)             x25519.rs:390-392 -> C/montgomery.rs:150-211   k_x25519       one thread per pair, the ladder
//                                                                                         of x25519.cuh on the FP64 field
//   PublicKey::from(&secret) x25519.rs:105-110 -> C/montgomery.rs:164-174   k_x25519_base  mul_base_clamped(k).to_montgomery()
//                            -> C/edwards.rs:580-590                                       as a constant-time fixed-base comb
//   EdwardsPoint::mul_base / mul_base_clamped   C/edwards.rs:918-957         k_x25519_base  the same comb, other encoders:
//   RistrettoPoint::mul_base                    C/ristretto.rs:939                          CompressedEdwardsY, CompressedRistretto
//   MontgomeryPoint::mul_base / mul_base_clamped C/montgomery.rs:143-174                    or Montgomery u; clamped or not
// Both are constant time in k and u: no branch, loop bound or address depends on them (x25519.cuh; comb.cuh scans
// every entry of a table row).  The comb table of the Ed25519 basepoint B (64 x 8 entries (j+1) 16^i B, 60 KiB) is
// built once per context.  Unlike base.cu's mul_base, which indexes its table by the digit, the comb never reads a
// secret-dependent address.
// The device workspaces that held scalars or shared secrets are cleared before a host-buffer call returns, as the
// reference zeroizes its secrets on drop (x25519.rs:112-117).
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "comb.cuh"
#include "engine.h"
#include "pieces.h"
#include "x25519.cuh"

static_assert(DALEK_POINTS_MONTGOMERY != DALEK_POINTS_COMPRESSED && DALEK_POINTS_MONTGOMERY != DALEK_POINTS_RISTRETTO, "formats");

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define X25519_THREADS 128
#define X25519_COMB_THREADS 384
#define X25519_COMB_DOUBLES COMB_BASE_DOUBLES

__global__ void __launch_bounds__(X25519_THREADS)
k_x25519(const uint32_t *__restrict__ scalars, const uint32_t *__restrict__ us, size_t n, uint32_t *__restrict__ out,
         uint8_t *__restrict__ contributory)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t k[8], u[8], r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { k[j] = scalars[8 * i + j]; u[j] = us[8 * i + j]; }
    x25519_ladder(r, k, u);
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
    if (contributory) contributory[i] = (uint8_t)x25519_contributory(r);
}

__global__ void __launch_bounds__(128) k_x25519_base_table(double *__restrict__ table)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 64 * 8) return;
    ge_p3 B; ge_p3_basepoint(B);
    comb_entry(table + (size_t)t * COMB_ENTRY, B, t >> 3, t & 7);
}

// s B for the scalar s of item i, encoded as OUT (DALEK_POINTS_COMPRESSED, _RISTRETTO or _MONTGOMERY): 64 mixed additions
// over the radix-16 signed digits of s, read as it is (CLAMP = 0, bit 255 clear: the value is not reduced, and since B
// has order l the point is (s mod l) B) or clamped (CLAMP = 1, clamp_integer, C/scalar.rs:1407-1412, not reduced).  Both
// keep s < 2^255, so the recoding of scalar.rs:1019-1051 holds.  Montgomery u = (Z + Y) / (Z - Y) (C/edwards.rs:580-590);
// the identity (s = 0 mod l) gives u = 0 like the reference's to_montgomery.
template <int OUT, int CLAMP>
__global__ void __launch_bounds__(X25519_COMB_THREADS, 1)
k_x25519_base(const uint32_t *__restrict__ scalars, const double *__restrict__ table, size_t n, uint32_t *__restrict__ out)
{
    extern __shared__ double s_tab[];                             // X25519_COMB_DOUBLES
    for (int k = threadIdx.x; k < X25519_COMB_DOUBLES; k += blockDim.x) s_tab[k] = table[k];
    __syncthreads();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge64_p3 acc;
    uint32_t w = 0;
    comb_mul_base_nibbles(acc, s_tab, [&](int pos) {
        if ((pos & 7) == 0) {                                     // one scalar word per 8 digits, clamped as it is read
            w = scalars[8 * i + (pos >> 3)];
            if (CLAMP) {
                w &= pos == 0 ? 0xfffffff8u : 0xffffffffu;
                w = pos == 56 ? ((w & 0x7fffffffu) | 0x40000000u) : w;
            }
        }
        const uint32_t v = w & 15;
        w >>= 4;
        return v;
    });
    uint32_t r[8];
    if (OUT == DALEK_POINTS_MONTGOMERY) {
        fe64 num, den, inv, u;
        fe64_add(num, acc.Z, acc.Y);                              // 2
        fe64_sub(den, acc.Z, acc.Y); fe64_carry(den, den);        // 1
        x25519_invert(inv, den);
        fe64_mul(u, num, inv);                                    // 2 x 1
        x25519_encode(r, u);
    } else {
        ge_p3 q; ge64_to_p3(q, acc);
        if (OUT == DALEK_POINTS_RISTRETTO) ristretto_compress<1>(r, q);
        else ge_compress<1>(r, q);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

template <int OUT, int CLAMP>
static int x25519_base_smem_attr(dalek_b200_ctx *ctx)
{
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_x25519_base<OUT, CLAMP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(X25519_COMB_DOUBLES * sizeof(double))));
    return 0;
}

// the comb table of B, built once per context (with the dynamic shared-memory limit of every k_x25519_base instance)
int comb_base_table_ensure(dalek_b200_ctx *ctx)
{
    if (ctx->comb_base_table_ready) return 0;
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_COMB_BASE_TABLE], X25519_COMB_DOUBLES * sizeof(double)))) return rc;
    if ((rc = x25519_base_smem_attr<DALEK_POINTS_MONTGOMERY, 1>(ctx)) || (rc = x25519_base_smem_attr<DALEK_POINTS_MONTGOMERY, 0>(ctx)) ||
        (rc = x25519_base_smem_attr<DALEK_POINTS_COMPRESSED, 1>(ctx)) || (rc = x25519_base_smem_attr<DALEK_POINTS_COMPRESSED, 0>(ctx)) ||
        (rc = x25519_base_smem_attr<DALEK_POINTS_RISTRETTO, 0>(ctx)))
        return rc;
    k_x25519_base_table<<<4, 128, 0, ctx->stream>>>((double *)ctx->ws[WS_COMB_BASE_TABLE].p);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->comb_base_table_ready = true;
    return 0;
}

static void launch_x25519(const void *d_k, const void *d_u, size_t m, void *d_out, void *d_contrib, cudaStream_t st)
{
    k_x25519<<<cdiv(m, X25519_THREADS), X25519_THREADS, 0, st>>>((const uint32_t *)d_k, (const uint32_t *)d_u, m,
                                                               (uint32_t *)d_out, (uint8_t *)d_contrib);
}

// one piece of the fixed-base comb: m scalars at d_k -> m encodings at d_out
static void launch_x25519_base(int out_fmt, bool clamp, const double *table, const void *d_k, size_t m, void *d_out, cudaStream_t st)
{
    const unsigned grid = cdiv(m, X25519_COMB_THREADS);
    const size_t smem = X25519_COMB_DOUBLES * sizeof(double);
    const uint32_t *k = (const uint32_t *)d_k;
    uint32_t *o = (uint32_t *)d_out;
    if (out_fmt == DALEK_POINTS_MONTGOMERY && clamp) k_x25519_base<DALEK_POINTS_MONTGOMERY, 1><<<grid, X25519_COMB_THREADS, smem, st>>>(k, table, m, o);
    else if (out_fmt == DALEK_POINTS_MONTGOMERY) k_x25519_base<DALEK_POINTS_MONTGOMERY, 0><<<grid, X25519_COMB_THREADS, smem, st>>>(k, table, m, o);
    else if (out_fmt == DALEK_POINTS_COMPRESSED && clamp) k_x25519_base<DALEK_POINTS_COMPRESSED, 1><<<grid, X25519_COMB_THREADS, smem, st>>>(k, table, m, o);
    else if (out_fmt == DALEK_POINTS_COMPRESSED) k_x25519_base<DALEK_POINTS_COMPRESSED, 0><<<grid, X25519_COMB_THREADS, smem, st>>>(k, table, m, o);
    else k_x25519_base<DALEK_POINTS_RISTRETTO, 0><<<grid, X25519_COMB_THREADS, smem, st>>>(k, table, m, o);
}

// the fixed-base comb over host buffers: the cached table of B, the batch streamed in pieces, the staging cleared
static int x25519_base_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, int out_fmt, bool clamp, uint8_t *out)
{
    int rc;
    if ((rc = comb_base_table_ensure(ctx))) return rc;
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    rc = run_pieces(ctx, nullptr, nullptr, scalars, 32, nullptr, 0, out, 32, nullptr, 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *dk, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st) {
                        launch_x25519_base(out_fmt, clamp, table, dk, m, d_o, st);
                        return 0;
                    });
    if (rc) return rc;
    return wipe_staging(ctx, n * 32, n * 32);
}

extern "C" {

int dalek_b200_x25519_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, const uint8_t *us, size_t n, uint8_t *out,
                            uint8_t *contributory)
{
    if (!ctx || (n && (!scalars || !us || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const size_t c_sz = contributory ? 1 : 0;
    int rc = run_pieces(ctx, nullptr, nullptr, scalars, 32, us, 32, out, 32, contributory, c_sz, n,
                        [&](const uint8_t *, const uint64_t *, const uint8_t *dk, const uint8_t *du, size_t m, uint8_t *d_o,
                            uint8_t *d_c, cudaStream_t st) {
                            launch_x25519(dk, du, m, d_o, c_sz ? d_c : nullptr, st);
                            return 0;
                        });
    if (rc) return rc;
    return wipe_staging(ctx, n * 64, n * (32 + c_sz));
}

int dalek_b200_x25519_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_us, size_t n, void *d_out,
                                void *d_contributory)
{
    if (!ctx || (n && (!d_scalars || !d_us || !d_out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    launch_x25519(d_scalars, d_us, n, d_out, d_contributory, ctx->stream);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = 1;
    return DALEK_OK;
}

int dalek_b200_x25519_public_keys(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!scalars || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return x25519_base_batch(ctx, scalars, n, DALEK_POINTS_MONTGOMERY, true, out);
}

int dalek_b200_mul_base_ct_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, int out_fmt, int flags, uint8_t *out)
{
    if (!ctx || (n && (!scalars || !out))) return DALEK_E_INVALID_ARG;
    if (out_fmt != DALEK_POINTS_COMPRESSED && out_fmt != DALEK_POINTS_RISTRETTO && out_fmt != DALEK_POINTS_MONTGOMERY) return DALEK_E_INVALID_ARG;
    if (flags & ~DALEK_MUL_CLAMPED) return DALEK_E_INVALID_ARG;
    const bool clamp = (flags & DALEK_MUL_CLAMPED) != 0;
    if (clamp && out_fmt == DALEK_POINTS_RISTRETTO) {
        ctx->last_error = "clamped multiplication is defined for Edwards and Montgomery points only";
        return DALEK_E_INVALID_ARG;
    }
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    if (!clamp) {                                                  // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear
        uint8_t top = 0;
        for (size_t i = 0; i < n; i++) top |= scalars[32 * i + 31];
        if (top & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    }
    CallTimer timer(ctx);
    return x25519_base_batch(ctx, scalars, n, out_fmt, clamp, out);
}

}  // extern "C"
