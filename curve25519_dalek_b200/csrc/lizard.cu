// lizard.cu -- Lizard encoding and decoding and the Ristretto Elligator map and its inverse in bulk: one thread per item
// over lizard.cuh, one kernel per entry point.
//   RistrettoPoint::map_to_curve            C/ristretto/elligator.rs:62-67     k_ristretto_map_to_curve    32 B -> CompressedRistretto
//   RistrettoPoint::lizard_encode::<Sha256> C/lizard/lizard_ristretto.rs:25-39 k_lizard_encode             16 B -> CompressedRistretto
//   RistrettoPoint::lizard_decode::<Sha256> :43-71                            k_lizard_decode<FMT>        point -> 16 B, status
//   RistrettoPoint::map_to_curve_inverse    :213-219                          k_map_to_curve_inverse<FMT> point -> 16 x 32 B, mask
// Points are CompressedRistretto or extended (20 radix-2^51 limbs, used exactly as given: the candidate order of the
// inverse depends on the representative).  Host buffers stream in pieces through run_pieces.  The payloads are
// plaintexts: every call clears the device copies of its staged inputs and outputs before it returns, also after a
// failed launch.  Constant time in the payloads and the points (lizard.cuh); a kernel branches only on its thread range.
#include <algorithm>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "lizard.cuh"
#include "pieces.h"
#include "point_load.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define LIZARD_THREADS 128

enum { LZ_SOME = 0, LZ_NONE = 1, LZ_UNDECODABLE = 2 };

__global__ void __launch_bounds__(LIZARD_THREADS)
k_ristretto_map_to_curve(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8], r[8];
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = in[8 * i + k];
    ristretto_map_to_curve(r, w);
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * i + k] = r[k];
}

__global__ void __launch_bounds__(LIZARD_THREADS)
k_lizard_encode(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t d[4], r[8];
#pragma unroll
    for (int k = 0; k < 4; k++) d[k] = in[4 * i + k];
    lizard_encode(r, d);
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * i + k] = r[k];
}

// status: LZ_SOME (payload in out), LZ_NONE (not exactly one candidate passes), LZ_UNDECODABLE; out is zero unless LZ_SOME
template <int FMT>
__global__ void __launch_bounds__(LIZARD_THREADS)
k_lizard_decode(const uint32_t *__restrict__ points, size_t n, uint32_t *__restrict__ out, uint8_t *__restrict__ status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 P;
    const uint32_t good = varmul_load_point<FMT>(P, points, i);
    uint32_t d[4];
    const uint32_t n_found = lizard_decode(d, P);
    const uint32_t gm = 0u - good;
#pragma unroll
    for (int k = 0; k < 4; k++) out[4 * i + k] = d[k] & gm;
    status[i] = (uint8_t)((good * (uint32_t)(n_found != 1)) | ((1u - good) * LZ_UNDECODABLE));
}

// out: 16 candidates of 32 bytes per item; mask: bit j set iff candidate j is Some.  An undecodable encoding gives
// zeros and mask 0, and sets *bad (one atomic per warp, whatever the points).
template <int FMT>
__global__ void __launch_bounds__(LIZARD_THREADS)
k_map_to_curve_inverse(const uint32_t *__restrict__ points, size_t n, uint4 *__restrict__ out, uint16_t *__restrict__ mask, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 P;
    const uint32_t good = varmul_load_point<FMT>(P, points, i);
    const uint32_t gm = 0u - good;
    uint4 *o = out + 32 * i;
    const uint32_t m = map_to_curve_inverse(P, [&](uint32_t j, const uint32_t b[8], uint32_t) {
        o[2 * j] = make_uint4(b[0] & gm, b[1] & gm, b[2] & gm, b[3] & gm);
        o[2 * j + 1] = make_uint4(b[4] & gm, b[5] & gm, b[6] & gm, b[7] & gm);
    });
    mask[i] = (uint16_t)(m & gm);
    const unsigned act = __activemask();
    const uint32_t any_bad = __reduce_or_sync(act, 1u - good);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicOr(bad, (int)any_bad);
}

// clear the staged inputs and outputs (the payloads are plaintexts), up to what the workspaces hold, then wait
static int lizard_wipe(dalek_b200_ctx *ctx, size_t in_bytes, size_t out_bytes)
{
    if (ctx->ws[WS_STAGING_IN].p) CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_IN].p, 0, std::min(in_bytes, ctx->ws[WS_STAGING_IN].cap), ctx->stream));
    if (ctx->ws[WS_STAGING_OUT].p) CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_OUT].p, 0, std::min(out_bytes, ctx->ws[WS_STAGING_OUT].cap), ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// a call's result: the first failure, else the wipe's
static int lizard_finish(dalek_b200_ctx *ctx, int rc, size_t in_bytes, size_t out_bytes)
{
    const int wrc = lizard_wipe(ctx, in_bytes, out_bytes);
    return rc ? rc : wrc;
}

static bool lizard_point_fmt_ok(int fmt) { return fmt == DALEK_POINTS_RISTRETTO || fmt == DALEK_POINTS_EXTENDED; }

extern "C" {

int dalek_b200_ristretto_map_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const int rc = run_pieces(ctx, nullptr, nullptr, in, 32, nullptr, 0, out, 32, nullptr, 0, n,
                              [&](const uint8_t *, const uint64_t *, const uint8_t *d_in, const uint8_t *, size_t m, uint8_t *d_o,
                                  uint8_t *, cudaStream_t st) {
                                  k_ristretto_map_to_curve<<<cdiv(m, LIZARD_THREADS), LIZARD_THREADS, 0, st>>>(
                                      (const uint32_t *)d_in, m, (uint32_t *)d_o);
                                  return 0;
                              });
    return lizard_finish(ctx, rc, n * 32, n * 32);
}

int dalek_b200_ristretto_lizard_encode_batch(dalek_b200_ctx *ctx, const uint8_t *data, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!data || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const int rc = run_pieces(ctx, nullptr, nullptr, data, 16, nullptr, 0, out, 32, nullptr, 0, n,
                              [&](const uint8_t *, const uint64_t *, const uint8_t *d_in, const uint8_t *, size_t m, uint8_t *d_o,
                                  uint8_t *, cudaStream_t st) {
                                  k_lizard_encode<<<cdiv(m, LIZARD_THREADS), LIZARD_THREADS, 0, st>>>((const uint32_t *)d_in, m,
                                                                                                     (uint32_t *)d_o);
                                  return 0;
                              });
    return lizard_finish(ctx, rc, n * 16, n * 32);
}

int dalek_b200_ristretto_lizard_decode_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n, uint8_t *data_out,
                                             uint8_t *status)
{
    if (!ctx || (n && (!points || !data_out || !status)) || !lizard_point_fmt_ok(point_fmt)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const size_t pin = msm_point_bytes(point_fmt);
    int rc = run_pieces(ctx, nullptr, nullptr, (const uint8_t *)points, pin, nullptr, 0, data_out, 16, status, 1, n,
                        [&](const uint8_t *, const uint64_t *, const uint8_t *d_p, const uint8_t *, size_t m, uint8_t *d_o,
                            uint8_t *d_s, cudaStream_t st) {
                            const unsigned g = cdiv(m, LIZARD_THREADS);
                            if (point_fmt == DALEK_POINTS_EXTENDED)
                                k_lizard_decode<DALEK_POINTS_EXTENDED><<<g, LIZARD_THREADS, 0, st>>>((const uint32_t *)d_p, m,
                                                                                                    (uint32_t *)d_o, d_s);
                            else
                                k_lizard_decode<DALEK_POINTS_RISTRETTO><<<g, LIZARD_THREADS, 0, st>>>((const uint32_t *)d_p, m,
                                                                                                     (uint32_t *)d_o, d_s);
                            return 0;
                        });
    if ((rc = lizard_finish(ctx, rc, n * pin, n * 17))) return rc;
    uint8_t any = 0;
    for (size_t i = 0; i < n; i++) any |= status[i];
    return any ? DALEK_NONE : DALEK_OK;
}

int dalek_b200_ristretto_map_to_curve_inverse_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n, uint8_t *out,
                                                    uint16_t *mask)
{
    if (!ctx || (n && (!points || !out || !mask)) || !lizard_point_fmt_ok(point_fmt)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], 64))) return rc;
    int *d_bad = (int *)ctx->ws[WS_CALL_SCRATCH].p;
    CUDA_TRY(ctx, cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
    const size_t pin = msm_point_bytes(point_fmt);
    rc = run_pieces(ctx, nullptr, nullptr, (const uint8_t *)points, pin, nullptr, 0, out, 512, (uint8_t *)mask, 2, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_p, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *d_m,
                        cudaStream_t st) {
                        const unsigned g = cdiv(m, LIZARD_THREADS);
                        if (point_fmt == DALEK_POINTS_EXTENDED)
                            k_map_to_curve_inverse<DALEK_POINTS_EXTENDED><<<g, LIZARD_THREADS, 0, st>>>(
                                (const uint32_t *)d_p, m, (uint4 *)d_o, (uint16_t *)d_m, d_bad);
                        else
                            k_map_to_curve_inverse<DALEK_POINTS_RISTRETTO><<<g, LIZARD_THREADS, 0, st>>>(
                                (const uint32_t *)d_p, m, (uint4 *)d_o, (uint16_t *)d_m, d_bad);
                        return 0;
                    });
    int bad = 0;
    if (!rc && !(rc = pinned_reserve(ctx, 64))) {
        if (cudaMemcpyAsync(ctx->h_pinned, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
    }
    if ((rc = lizard_finish(ctx, rc, n * pin, n * 514))) return rc;
    bad = *(const int *)ctx->h_pinned;
    return bad ? DALEK_NONE : DALEK_OK;
}

}  // extern "C"
