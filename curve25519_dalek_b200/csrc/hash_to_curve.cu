// hash_to_curve.cu -- hashing into the group in bulk: one thread per item over the maps of elligator.cuh.
//   RistrettoPoint::from_uniform_bytes     C/ristretto.rs:774-790   k_ristretto_from_uniform   64 B -> CompressedRistretto
//   RistrettoPoint::hash_from_bytes        C/ristretto.rs:736-761   k_ristretto_hash_bytes     message -> CompressedRistretto
//   EdwardsPoint::hash_to_curve            C/edwards.rs:736-750     k_edwards_h2c<2>           message, DST -> CompressedEdwardsY
//   EdwardsPoint::encode_to_curve          C/edwards.rs:710-721     k_edwards_h2c<1>
// Host buffers stream in pieces over the context's two streams: the 64-byte inputs through run_pieces, the flat
// messages the way ed25519_b200_verify_each_flat does (each piece copies its byte range and its offsets).  The DST (one
// per call, at most 255 bytes) travels as a __grid_constant__ kernel parameter.
#include <algorithm>

#include "../../include/dalek_b200.h"
#include "elligator.cuh"
#include "engine.h"
#include "pieces.h"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define H2C_THREADS 128

struct H2cDst {
    uint8_t b[256];
    uint32_t len;
};

__global__ void __launch_bounds__(H2C_THREADS)
k_ristretto_from_uniform(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[16], r[8];
#pragma unroll
    for (int j = 0; j < 16; j++) w[j] = in[16 * i + j];
    ge_p3 P;
    ristretto_from_uniform(P, w);
    ristretto_compress<1>(r, P);
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

// msgs: the whole flat buffer (offsets are absolute); offs: this piece's n + 1 offsets
__global__ void __launch_bounds__(H2C_THREADS)
k_ristretto_hash_bytes(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, size_t n, uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t o0 = offs[i], o1 = offs[i + 1];
    uint32_t r[8];
    ristretto_hash_from_bytes(r, msgs + o0, (size_t)(o1 - o0));
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

template <int COUNT>
__global__ void __launch_bounds__(H2C_THREADS)
k_edwards_h2c(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, size_t n, const __grid_constant__ H2cDst dst,
              uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t o0 = offs[i], o1 = offs[i + 1];
    uint32_t r[8];
    edwards_hash_to_curve<COUNT>(r, msgs + o0, (size_t)(o1 - o0), dst.b, dst.len);
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

// the flat-message calls: offsets start at 0 and do not decrease (ed25519_b200_verify_each_flat, single.cu:407-412)
static bool offsets_ok(const uint64_t *offs, size_t n)
{
    if (offs[0] != 0) return false;
    for (size_t i = 0; i < n; i++)
        if (offs[i] > offs[i + 1]) return false;
    return true;
}

// count = 0: hash_from_bytes; 1: encode_to_curve; 2: hash_to_curve
static int run_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n, const H2cDst *dst,
                    int count, uint8_t *out)
{
    int rc;
    const size_t mbytes = (size_t)msg_offsets[n];
    if ((rc = ws_reserve(ctx, ctx->misc1, mbytes + 16))) return rc;
    if ((rc = ws_reserve(ctx, ctx->msg_offs, (n + 1) * 8))) return rc;
    if ((rc = ws_reserve(ctx, ctx->points, n * 32))) return rc;
    uint8_t *d_msgs = (uint8_t *)ctx->misc1.p, *d_out = (uint8_t *)ctx->points.p;
    uint64_t *d_offs = (uint64_t *)ctx->msg_offs.p;
    cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    const size_t piece = n >= (1u << 17) ? (size_t)1 << 16 : n;
    size_t k = 0;
    for (size_t lo = 0; lo < n; lo += piece, k++) {
        const size_t m = std::min(piece, n - lo);
        cudaStream_t st = ss[k & 1];
        const size_t m0 = (size_t)msg_offsets[lo], m1 = (size_t)msg_offsets[lo + m];
        if (m1 > m0) CUDA_TRY(ctx, cudaMemcpyAsync(d_msgs + m0, msgs_flat + m0, m1 - m0, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_offs + lo, msg_offsets + lo, (m + 1) * 8, cudaMemcpyHostToDevice, st));
        uint32_t *o = (uint32_t *)(d_out + lo * 32);
        if (count == 0) k_ristretto_hash_bytes<<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs + lo, m, o);
        else if (count == 1) k_edwards_h2c<1><<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs + lo, m, *dst, o);
        else k_edwards_h2c<2><<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs + lo, m, *dst, o);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(out + lo * 32, d_out + lo * 32, m * 32, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)k;
    return DALEK_OK;
}

static int edwards_h2c(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n, const uint8_t *dst,
                       size_t dst_len, uint8_t *out, int count)
{
    if (!ctx || (n && (!msgs_flat || !msg_offsets || !out)) || !dst || dst_len == 0 || dst_len > 255) return DALEK_E_INVALID_ARG;
    if (n && !offsets_ok(msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    H2cDst d = {};
    for (size_t j = 0; j < dst_len; j++) d.b[j] = dst[j];
    d.len = (uint32_t)dst_len;
    return run_flat(ctx, msgs_flat, msg_offsets, n, &d, count, out);
}

extern "C" {

int dalek_b200_ristretto_from_uniform_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_pieces(ctx, in, 64, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *d_in, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *, cudaStream_t st) {
                          k_ristretto_from_uniform<<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>((const uint32_t *)d_in, m,
                                                                                                (uint32_t *)d_o);
                      });
}

int dalek_b200_ristretto_hash_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                               size_t n, uint8_t *out)
{
    if (!ctx || (n && (!msgs_flat || !msg_offsets || !out))) return DALEK_E_INVALID_ARG;
    if (n && !offsets_ok(msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_flat(ctx, msgs_flat, msg_offsets, n, nullptr, 0, out);
}

int dalek_b200_edwards_hash_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n,
                                           const uint8_t *dst, size_t dst_len, uint8_t *out)
{
    return edwards_h2c(ctx, msgs_flat, msg_offsets, n, dst, dst_len, out, 2);
}

int dalek_b200_edwards_encode_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n,
                                             const uint8_t *dst, size_t dst_len, uint8_t *out)
{
    return edwards_h2c(ctx, msgs_flat, msg_offsets, n, dst, dst_len, out, 1);
}

}  // extern "C"
