// hash_to_curve.cu -- hashing into the group in bulk: one thread per item over the maps of elligator.cuh.
//   RistrettoPoint::from_uniform_bytes     C/ristretto.rs:774-790   k_ristretto_from_uniform   64 B -> CompressedRistretto
//   RistrettoPoint::hash_from_bytes        C/ristretto.rs:736-761   k_ristretto_hash_bytes     message -> CompressedRistretto
//   EdwardsPoint::hash_to_curve            C/edwards.rs:736-750     k_edwards_h2c<2>           message, DST -> CompressedEdwardsY
//   EdwardsPoint::encode_to_curve          C/edwards.rs:710-721     k_edwards_h2c<1>
// Host buffers stream in pieces over the context's two streams through run_pieces (each piece of flat messages copies
// its byte range and its offsets).  The DST (one per call, at most 255 bytes) travels as a __grid_constant__ kernel
// parameter.
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

// count = 1: encode_to_curve; 2: hash_to_curve
static int edwards_h2c(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n, const uint8_t *dst,
                       size_t dst_len, uint8_t *out, int count)
{
    if (!ctx || (n && !out) || !flat_messages_ok(msgs_flat, msg_offsets, n) || !dst || dst_len == 0 || dst_len > 255)
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    H2cDst d = {};
    for (size_t j = 0; j < dst_len; j++) d.b[j] = dst[j];
    d.len = (uint32_t)dst_len;
    return run_pieces(ctx, msgs_flat, msg_offsets, nullptr, 0, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *, const uint8_t *, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st) {
                          uint32_t *o = (uint32_t *)d_o;
                          if (count == 1) k_edwards_h2c<1><<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs, m, d, o);
                          else k_edwards_h2c<2><<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs, m, d, o);
                          return 0;
                      });
}

extern "C" {

int dalek_b200_ristretto_from_uniform_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_pieces(ctx, nullptr, nullptr, in, 64, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *, const uint64_t *, const uint8_t *d_in, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                          cudaStream_t st) {
                          k_ristretto_from_uniform<<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>((const uint32_t *)d_in, m,
                                                                                                (uint32_t *)d_o);
                          return 0;
                      });
}

int dalek_b200_ristretto_hash_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                               size_t n, uint8_t *out)
{
    if (!ctx || (n && !out) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_pieces(ctx, msgs_flat, msg_offsets, nullptr, 0, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *, const uint8_t *, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st) {
                          k_ristretto_hash_bytes<<<cdiv(m, H2C_THREADS), H2C_THREADS, 0, st>>>(d_msgs, d_offs, m, (uint32_t *)d_o);
                          return 0;
                      });
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
