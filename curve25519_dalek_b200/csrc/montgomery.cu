// montgomery.cu -- batched MontgomeryPoint arithmetic (C/montgomery.rs) beyond X25519:
//   Scalar * MontgomeryPoint      C/montgomery.rs:484-505   k_mont_ladder<8>      the ladder of x25519.cuh over bits 254..0
//                                                                                 of the unclamped Scalar
//   MontgomeryPoint::mul_bits_be  C/montgomery.rs:176-211   k_mont_ladder<8|16>   the same ladder over bits nbits-1..0 of
//                                                                                 an integer of up to 512 bits
//   MontgomeryPoint::to_edwards   C/montgomery.rs:223-268   k_mont_to_edwards     y = (u - 1) / (u + 1), then
//                                                                                 CompressedEdwardsY::decompress
// mul_clamped is x25519 (x25519.cu); mul_base / mul_base_clamped are the fixed-base comb of x25519.cu.
// The ladders are constant time in the integers and in u (x25519.cuh): one thread per item, nbits public and uniform per
// call, the integer's bytes read at addresses and under predicates that depend only on the public int_bytes.  The one
// exception is the report of a scalar with bit 255 set by the device-buffer call, which fails the call.  Host-buffer
// calls clear the device copies of the integers and of the results before they return.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "pieces.h"
#include "x25519.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define MONT_THREADS 128

// staging in WS_CALL_SCRATCH: status word, the broadcast integer (up to 64 bytes), the broadcast u
#define MT_STATUS 0
#define MT_INT 64
#define MT_U 128
#define MT_BYTES 256

enum { MT_BAD_SCALAR = 1, MT_NONE = 2 };

// out[i] = u([b_i] P_i), b_i = bits nbits-1..0 of the int_bytes-byte little-endian integer at ints + i_step i, u(P_i) the
// eight words at us + 8 u_step i (steps 0: item 0 for every item).  NW words hold the integer (nbits <= 32 NW); bytes
// past int_bytes read as 0.  check_top: report an integer with bit 255 set in *status (Scalar invariant #1).
// Minimum one block per SM: with the default bound ptxas holds the kernel to 168 registers and spills one of them across
// the ladder loop; without it the kernel takes ~250 registers and no stack, at the two blocks per SM of k_x25519.
template <int NW>
__global__ void __launch_bounds__(MONT_THREADS, 1)
k_mont_ladder(const uint8_t *__restrict__ ints, size_t i_step, int int_bytes, int nbits, const uint32_t *__restrict__ us,
              size_t u_step, size_t n, uint32_t *__restrict__ out, int check_top, int *status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *src = ints + i_step * i;
    uint32_t k[NW], u[8], r[8];
#pragma unroll
    for (int j = 0; j < NW; j++) k[j] = 0;
#pragma unroll
    for (int j = 0; j < 4 * NW; j++)
        if (j < int_bytes) k[j >> 2] |= (uint32_t)src[j] << (8 * (j & 3));
    if (check_top) {
        const uint32_t top = __reduce_or_sync(__activemask(), k[7] >> 31);
        if (top && (threadIdx.x & 31) == (uint32_t)(__ffs(__activemask()) - 1)) atomicOr(status, MT_BAD_SCALAR);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) u[j] = us[8 * (u_step * i) + j];
    mont_ladder<NW>(r, k, nbits, u);
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

// to_edwards(u_i, signs[i]) as CompressedEdwardsY; None (u = -1, or y not on the curve: u of the twist) gives ok = 0 and
// the identity's encoding.  The map is computed with one inversion as the reference does, so y is its canonical value.
__global__ void __launch_bounds__(MONT_THREADS)
k_mont_to_edwards(const uint32_t *__restrict__ us, const uint8_t *__restrict__ signs, size_t n, uint32_t *__restrict__ out,
                  uint8_t *__restrict__ ok, int *status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
#pragma unroll
    for (int j = 0; j < 8; j++) w[j] = us[8 * i + j];
    fe u, one, num, den, inv, y;
    fe_frombytes_words(u, w);                                    // bit 255 ignored (FieldElement::from_bytes)
    fe_1(one);
    fe_sub(num, u, one); fe_carry(num, num);                     // u - 1
    fe_add(den, u, one); fe_carry(den, den);                     // u + 1
    const uint32_t minus_one = (uint32_t)fe_iszero(den);        // u == -1 (montgomery.rs:254-256)
    fe_invert_f64(inv, den);
    fe_mul(y, num, inv);
    uint32_t yb[8];
    fe_tobytes_words(yb, y);                                     // y.to_bytes()
    yb[7] ^= (uint32_t)(signs[i] & 1u) << 31;                    // y_bytes[31] ^= sign << 7 (u8: bit 0 of sign only)
    fe x, yd;
    const uint32_t good = ge_decompress_affine<1>(x, yd, yb) & (1u - minus_one);
    uint32_t enc[8];
    fe_tobytes_words(enc, yd);                                   // compress: canonical y with the sign of x
    enc[7] ^= (uint32_t)fe_isnegative(x) << 31;
    const uint32_t keep = 0u - good;
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = (enc[j] & keep) | ((j == 0 ? 1u : 0u) & ~keep);
    if (ok) ok[i] = (uint8_t)good;
    if (!good) atomicOr(status, MT_NONE);                        // u is public
}

// one ladder launch of m items; i_step is int_bytes or 0, u_step 1 or 0 (broadcast of item 0)
static void mont_launch(const void *ints, size_t i_step, int int_bytes, int nbits, const void *us, size_t u_step, size_t m,
                        void *out, int check_top, int *status, cudaStream_t st)
{
    if (nbits <= 256)
        k_mont_ladder<8><<<cdiv(m, MONT_THREADS), MONT_THREADS, 0, st>>>((const uint8_t *)ints, i_step, int_bytes, nbits,
                                                                         (const uint32_t *)us, u_step, m, (uint32_t *)out,
                                                                         check_top, status);
    else
        k_mont_ladder<16><<<cdiv(m, MONT_THREADS), MONT_THREADS, 0, st>>>((const uint8_t *)ints, i_step, int_bytes, nbits,
                                                                          (const uint32_t *)us, u_step, m, (uint32_t *)out,
                                                                          check_top, status);
}

static int mont_read_status(dalek_b200_ctx *ctx, const int *d_status, int *status)
{
    int rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *status = *(const int *)ctx->h_pinned;
    return 0;
}

// the ladder over host buffers (arguments already checked, n > 0): broadcast items staged in WS_CALL_SCRATCH, the rest
// streamed in pieces with u first (word-aligned) and the integers second (read bytewise, any int_bytes)
static int mont_ladder_host(dalek_b200_ctx *ctx, const uint8_t *ints, size_t int_bytes, size_t n_ints, int nbits, const uint8_t *us,
                            size_t n_points, size_t n, uint8_t *out)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], MT_BYTES))) return rc;
    char *base = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    const bool bi = n_ints == 1, bu = n_points == 1;
    if (bi) CUDA_TRY(ctx, cudaMemcpyAsync(base + MT_INT, ints, int_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (bu) CUDA_TRY(ctx, cudaMemcpyAsync(base + MT_U, us, 32, cudaMemcpyHostToDevice, ctx->stream));
    const size_t i_sz = bi ? 0 : int_bytes, u_sz = bu ? 0 : 32;
    rc = run_pieces(ctx, nullptr, nullptr, bu ? nullptr : us, u_sz, bi ? nullptr : ints, i_sz, out, 32, nullptr, 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_u, const uint8_t *d_i, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st) {
                        mont_launch(bi ? base + MT_INT : (const char *)d_i, bi ? 0 : int_bytes, (int)int_bytes, nbits,
                                    bu ? base + MT_U : (const char *)d_u, bu ? 0 : 1, m, d_o, 0, nullptr, st);
                        return 0;
                    });
    if (rc) return rc;
    CUDA_TRY(ctx, cudaMemsetAsync(base + MT_INT, 0, 64, ctx->stream));            // zeroize on drop
    return wipe_staging(ctx, n * (i_sz + u_sz), n * 32);
}

static int broadcast_ok(dalek_b200_ctx *ctx, size_t n_a, size_t n_b, size_t n)
{
    if ((n_a != 1 && n_a != n) || (n_b != 1 && n_b != n)) {
        ctx->last_error = "each input count must be 1 or n";
        return 0;
    }
    return 1;
}

extern "C" {

int dalek_b200_montgomery_mul_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n_scalars, const uint8_t *us,
                                    size_t n_points, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!scalars || !us || !out))) return DALEK_E_INVALID_ARG;
    if (!broadcast_ok(ctx, n_scalars, n_points, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    uint8_t top = 0;                                               // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear
    for (size_t i = 0; i < n_scalars; i++) top |= scalars[32 * i + 31];
    if (top & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    CallTimer timer(ctx);
    return mont_ladder_host(ctx, scalars, 32, n_scalars, 255, us, n_points, n, out);
}

int dalek_b200_montgomery_mul_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, size_t n_scalars, const void *d_us,
                                        size_t n_points, size_t n, void *d_out)
{
    if (!ctx || (n && (!d_scalars || !d_us || !d_out))) return DALEK_E_INVALID_ARG;
    if (!broadcast_ok(ctx, n_scalars, n_points, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], MT_BYTES))) return rc;
    int *d_status = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + MT_STATUS);
    CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    mont_launch(d_scalars, n_scalars == 1 ? 0 : 32, 32, 255, d_us, n_points == 1 ? 0 : 1, n, d_out, 1, d_status, ctx->stream);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    int status = 0;
    if ((rc = mont_read_status(ctx, d_status, &status))) return rc;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = 1;
    if (status & MT_BAD_SCALAR) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    return DALEK_OK;
}

int dalek_b200_montgomery_mul_bits_be_batch(dalek_b200_ctx *ctx, const uint8_t *ints, size_t int_bytes, size_t n_ints,
                                            size_t nbits, const uint8_t *us, size_t n_points, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!ints || !us || !out))) return DALEK_E_INVALID_ARG;
    if (int_bytes < 1 || int_bytes > 64 || nbits > 8 * int_bytes) {
        ctx->last_error = "int_bytes must be 1..64 and nbits at most 8 int_bytes";
        return DALEK_E_INVALID_ARG;
    }
    if (!broadcast_ok(ctx, n_ints, n_points, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return mont_ladder_host(ctx, ints, int_bytes, n_ints, (int)nbits, us, n_points, n, out);
}

int dalek_b200_montgomery_to_edwards_batch(dalek_b200_ctx *ctx, const uint8_t *us, const uint8_t *signs, size_t n, uint8_t *out,
                                           uint8_t *ok)
{
    if (!ctx || (n && (!us || !signs || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], MT_BYTES))) return rc;
    int *d_status = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + MT_STATUS);
    CUDA_TRY(ctx, cudaMemsetAsync(d_status, 0, 4, ctx->stream));
    const size_t ok_sz = ok ? 1 : 0;
    rc = run_pieces(ctx, nullptr, nullptr, us, 32, signs, 1, out, 32, ok, ok_sz, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_u, const uint8_t *d_s, size_t m, uint8_t *d_o, uint8_t *d_ok,
                        cudaStream_t st) {
                        k_mont_to_edwards<<<cdiv(m, MONT_THREADS), MONT_THREADS, 0, st>>>((const uint32_t *)d_u, d_s, m, (uint32_t *)d_o,
                                                                                         ok_sz ? d_ok : nullptr, d_status);
                        return 0;
                    });
    if (rc) return rc;
    int status = 0;
    if ((rc = mont_read_status(ctx, d_status, &status))) return rc;
    return (status & MT_NONE) ? DALEK_NONE : DALEK_OK;
}

}  // extern "C"
