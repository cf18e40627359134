// double_base.cu -- batched variable-time double-base scalar multiplication out[i] = a_i A_i + b_i B, B the basepoint:
//   EdwardsPoint::vartime_double_scalar_mul_basepoint    C/edwards.rs:1078-1087 -> vartime_double_base.rs:23-72
//   RistrettoPoint::vartime_double_scalar_mul_basepoint  C/ristretto.rs:1051-1063
// k_vartime_double_base: one thread per item.  It decodes A_i (point_load.cuh), runs double_base.cuh with A_i's 8-entry
// table in local memory and B's 8 entries (row 0 of WS_BASE_TABLE) in shared memory, and encodes the result.  The
// scalars are used as given, not reduced: A_i may carry a torsion component, and then a A_i != (a mod l) A_i.
// Variable time: scalars and points are public, so no staged copy is cleared.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "double_base.cuh"
#include "engine.h"
#include "pieces.h"
#include "point_load.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define DB_THREADS 128

enum { DB_BAD_POINT = 1, DB_BAD_SCALAR = 2 };

template <int FMT>
__device__ __forceinline__ void db_encode(uint32_t *__restrict__ out, const ge64_p3 &Q)
{
    ge_p3 q; ge64_to_p3(q, Q);
    uint32_t w[8];
    if (FMT == DALEK_POINTS_RISTRETTO) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
#pragma unroll
    for (int k = 0; k < 8; k++) out[k] = w[k];
}

// ab: n pairs a_i || b_i of 32-byte scalars; points: n points in format FMT
template <int FMT>
__global__ void __launch_bounds__(DB_THREADS, 2)
k_vartime_double_base(const uint32_t *__restrict__ ab, const uint32_t *__restrict__ points, size_t n,
                      const ge_niels_packed *__restrict__ base_row0, uint32_t *__restrict__ out, uint8_t *__restrict__ ok, int *status)
{
    __shared__ double s_B[8 * 15];                               // (j+1) B as balanced FP64 affine Niels, j = 0..7
    if (threadIdx.x < 8) double_base_stage_B(s_B + 15 * threadIdx.x, base_row0[threadIdx.x]);
    __syncthreads();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t a[8], b[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { a[k] = ab[16 * i + k]; b[k] = ab[16 * i + 8 + k]; }
    // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear.  A set bit fails the call; it is cleared here only to keep
    // the top digit inside the tables.
    const uint32_t top = __reduce_or_sync(__activemask(), (a[7] | b[7]) >> 31);
    if (top && (threadIdx.x & 31) == (uint32_t)(__ffs(__activemask()) - 1)) atomicOr(status, DB_BAD_SCALAR);
    a[7] &= 0x7fffffffu; b[7] &= 0x7fffffffu;
    ge_p3 p;
    const uint32_t good = varmul_load_point<FMT>(p, points, i);
    ge64_p3 Q;
    DoubleBaseLocal w;
    double_base_eval(Q, p, a, b, s_B, w);
    if (!good) ge64_identity(Q);                                  // an undecodable point's slot holds the identity
    db_encode<FMT>(out + 8 * i, Q);
    if (ok) ok[i] = (uint8_t)good;
    if (!good) atomicOr(status, DB_BAD_POINT);
}

static void db_launch(int fmt, const void *ab, const void *pts, size_t m, const ge_niels_packed *base, void *out, void *ok, int *status,
                      cudaStream_t st)
{
    const unsigned g = cdiv(m, DB_THREADS);
    if (fmt == DALEK_POINTS_EXTENDED)
        k_vartime_double_base<DALEK_POINTS_EXTENDED><<<g, DB_THREADS, 0, st>>>((const uint32_t *)ab, (const uint32_t *)pts, m, base,
                                                                               (uint32_t *)out, (uint8_t *)ok, status);
    else if (fmt == DALEK_POINTS_RISTRETTO)
        k_vartime_double_base<DALEK_POINTS_RISTRETTO><<<g, DB_THREADS, 0, st>>>((const uint32_t *)ab, (const uint32_t *)pts, m, base,
                                                                                (uint32_t *)out, (uint8_t *)ok, status);
    else
        k_vartime_double_base<DALEK_POINTS_COMPRESSED><<<g, DB_THREADS, 0, st>>>((const uint32_t *)ab, (const uint32_t *)pts, m, base,
                                                                                 (uint32_t *)out, (uint8_t *)ok, status);
}

static inline bool db_fmt_ok(int f)
{
    return f == DALEK_POINTS_COMPRESSED || f == DALEK_POINTS_EXTENDED || f == DALEK_POINTS_RISTRETTO;
}

// B's table and a cleared status word in WS_CALL_SCRATCH
static int db_setup(dalek_b200_ctx *ctx, int **status)
{
    int rc;
    if ((rc = base_table_ensure(ctx))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], 64))) return rc;
    *status = (int *)ctx->ws[WS_CALL_SCRATCH].p;
    CUDA_TRY(ctx, cudaMemsetAsync(*status, 0, 4, ctx->stream));
    return 0;
}

static int db_read_status(dalek_b200_ctx *ctx, const int *d_status, int *status)
{
    int rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *status = *(const int *)ctx->h_pinned;
    return 0;
}

extern "C" {

int dalek_b200_vartime_double_base_batch(dalek_b200_ctx *ctx, const uint8_t *ab, const void *points, int point_fmt, size_t n,
                                         uint8_t *out, uint8_t *ok)
{
    if (!ctx || (n && (!ab || !points || !out)) || !db_fmt_ok(point_fmt)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    uint8_t top = 0;                                               // Scalar invariant #1, before any device work
    for (size_t i = 0; i < 2 * n; i++) top |= ab[32 * i + 31];
    if (top & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    CallTimer timer(ctx);
    int *d_status, rc;
    if ((rc = db_setup(ctx, &d_status))) return rc;
    const ge_niels_packed *base = (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p;
    rc = run_pieces(ctx, nullptr, nullptr, ab, 64, (const uint8_t *)points, msm_point_bytes(point_fmt), out, 32, ok, ok ? 1 : 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_ab, const uint8_t *d_p, size_t m, uint8_t *d_o, uint8_t *d_ok,
                        cudaStream_t st) {
                        db_launch(point_fmt, d_ab, d_p, m, base, d_o, ok ? d_ok : nullptr, d_status, st);
                        return 0;
                    });
    if (rc) return rc;
    int status = 0;
    if ((rc = db_read_status(ctx, d_status, &status))) return rc;
    return (status & DB_BAD_POINT) ? DALEK_NONE : DALEK_OK;
}

int dalek_b200_vartime_double_base_batch_dev(dalek_b200_ctx *ctx, const void *d_ab, const void *d_points, int point_fmt, size_t n,
                                             void *d_out, void *d_ok)
{
    if (!ctx || (n && (!d_ab || !d_points || !d_out)) || !db_fmt_ok(point_fmt)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int *d_status, rc;
    if ((rc = db_setup(ctx, &d_status))) return rc;
    const ge_niels_packed *base = (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p;
    const size_t pin = msm_point_bytes(point_fmt);
    const size_t piece = n >= (1u << 17) ? (size_t)1 << 16 : n;     // the pieces of run_pieces
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    int k = 0;
    for (size_t lo = 0; lo < n; lo += piece, k++) {
        const size_t m = std::min(piece, n - lo);
        db_launch(point_fmt, (const uint8_t *)d_ab + 64 * lo, (const uint8_t *)d_points + pin * lo, m, base, (uint8_t *)d_out + 32 * lo,
                  d_ok ? (uint8_t *)d_ok + lo : nullptr, d_status, ctx->stream);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    int status = 0;
    if ((rc = db_read_status(ctx, d_status, &status))) return rc;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = k;
    if (status & DB_BAD_SCALAR) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    return (status & DB_BAD_POINT) ? DALEK_NONE : DALEK_OK;
}

}  // extern "C"
