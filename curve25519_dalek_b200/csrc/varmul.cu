// varmul.cu -- batched variable-base scalar multiplication out[i] = s_i P_i and the torsion checks of Edwards points.
//   EdwardsPoint * Scalar           C/edwards.rs:890-899 -> variable_base.rs:11-48   k_varmul       one thread per item
//   EdwardsPoint::mul_clamped       C/edwards.rs:932-941                               (clamped, not reduced)
//   RistrettoPoint * Scalar         C/ristretto.rs:917-926
//   BasepointTable::create(P) * s   C/edwards.rs:1140-1230, C/ristretto.rs:1086-1103  k_varmul_comb  one shared point
//   is_small_order / is_torsion_free C/edwards.rs:1405-1437                           k_torsion
// k_varmul decodes P_i, runs varmul.cuh on the FP64 field with its [P..8P] table in local memory, and encodes the
// result.  When one point serves a batch of at least VARMUL_COMB_MIN items, its 64 x 8 comb table (comb.cuh) is built
// once per call and every item costs 64 mixed additions and no doubling; both paths give the same bytes.
// Constant time in the scalars: no branch, loop bound or address depends on them (varmul.cuh; comb.cuh scans every
// entry of a table row).  The one exception is the report of a scalar with bit 255 set by a device-buffer call, which
// fails the call.  Host-buffer calls clear the device copies of the scalars and of the results before they return.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "comb.cuh"
#include "engine.h"
#include "pieces.h"
#include "point_load.cuh"
#include "varmul.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define VARMUL_THREADS 128
#define VARMUL_COMB_THREADS 384
#define VARMUL_COMB_MIN 16384         // shared-point batches from this size use the comb (measured, DESIGN.md §6)

// staging in WS_CALL_SCRATCH: status word, the broadcast scalar, the broadcast point, the comb table
#define VM_STATUS 0
#define VM_SCALAR 64
#define VM_POINT 128
#define VM_TABLE 512

enum { VM_BAD_POINT = 1, VM_BAD_SCALAR = 2 };

template <int FMT>
__device__ __forceinline__ void varmul_encode(uint32_t *__restrict__ out, const ge64_p3 &Q)
{
    ge_p3 q; ge64_to_p3(q, Q);
    uint32_t w[8];
    if (FMT == DALEK_POINTS_RISTRETTO) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
#pragma unroll
    for (int k = 0; k < 8; k++) out[k] = w[k];
}

// the scalar of item i (s_step 0: one scalar for all), clamped (clamp_integer, C/scalar.rs:1407-1412) or checked for
// bit 255 (Scalar invariant #1)
__device__ __forceinline__ void varmul_load_scalar(uint32_t s[8], const uint32_t *__restrict__ scalars, size_t s_step, size_t i,
                                                   uint32_t clamp, int *status)
{
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = scalars[8 * (s_step * i) + k];
    if (clamp) x25519_clamp(s);
    const uint32_t top = __reduce_or_sync(__activemask(), s[7] >> 31);
    if (top && (threadIdx.x & 31) == (uint32_t)(__ffs(__activemask()) - 1)) atomicOr(status, VM_BAD_SCALAR);
}

template <int FMT>
__global__ void __launch_bounds__(VARMUL_THREADS)
k_varmul(const uint32_t *__restrict__ scalars, size_t s_step, const uint32_t *__restrict__ points, size_t p_step, size_t n,
         uint32_t clamp, uint32_t *__restrict__ out, uint8_t *__restrict__ ok, int *status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    varmul_load_scalar(s, scalars, s_step, i, clamp, status);
    ge_p3 p;
    const uint32_t good = varmul_load_point<FMT>(p, points, p_step * i);
    ge64_p3 P, Q;
    ge64_from_p3(P, p);
    VarmulLocalTab tab;
    varmul(Q, s, P, tab);
    varmul_encode<FMT>(out + 8 * i, Q);
    if (ok) ok[i] = (uint8_t)good;
    if (!good) atomicOr(status, VM_BAD_POINT);                     // the point is public
}

// the comb table of the one point (entry (j+1) 16^i P, comb.cuh)
template <int FMT>
__global__ void __launch_bounds__(128) k_varmul_comb_table(const uint32_t *__restrict__ point, double *__restrict__ table, int *status)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 64 * 8) return;
    ge_p3 P;
    if (!varmul_load_point<FMT>(P, point, 0) && t == 0) atomicOr(status, VM_BAD_POINT);
    comb_entry(table + (size_t)t * COMB_ENTRY, P, t >> 3, t & 7);
}

template <int FMT>
__global__ void __launch_bounds__(VARMUL_COMB_THREADS, 1)
k_varmul_comb(const uint32_t *__restrict__ scalars, size_t s_step, const double *__restrict__ table, size_t n, uint32_t clamp,
              uint32_t *__restrict__ out, uint8_t *__restrict__ ok, int *status)
{
    extern __shared__ double s_tab[];                             // COMB_BASE_DOUBLES
    for (int k = threadIdx.x; k < COMB_BASE_DOUBLES; k += blockDim.x) s_tab[k] = table[k];
    __syncthreads();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    varmul_load_scalar(s, scalars, s_step, i, clamp, status);
    ge64_p3 Q;
    comb_mul_base(Q, s, s_tab);
    varmul_encode<FMT>(out + 8 * i, Q);
    if (ok) ok[i] = (uint8_t)((*status & VM_BAD_POINT) == 0);   // written by the table kernel before this launch
}

// flags: is_small_order | is_torsion_free << 1 | decoded << 2; 0 for an undecodable point
template <int FMT>
__global__ void __launch_bounds__(VARMUL_THREADS) k_torsion(const uint32_t *__restrict__ points, size_t n, uint8_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 p;
    const uint32_t good = varmul_load_point<FMT>(p, points, i);
    ge64_p3 P;
    ge64_from_p3(P, p);
    VarmulLocalTab tab;
    const uint32_t f = varmul_torsion_flags(P, tab) | 4u;
    out[i] = (uint8_t)(good ? f : 0u);
}

// how one call runs: the format, the path, the clamp flag and its device status word / comb table
struct VarmulPlan {
    int fmt;
    bool comb;
    uint32_t clamp;
    const double *table;
    int *status;
};

// one launch of m items; s_step / p_step are 1, or 0 to broadcast item 0's scalar / point
template <int FMT>
static void varmul_launch_fmt(const VarmulPlan &pl, const void *s, size_t s_step, const void *p, size_t p_step, size_t m, void *out,
                              void *ok, cudaStream_t st)
{
    if (pl.comb)
        k_varmul_comb<FMT><<<cdiv(m, VARMUL_COMB_THREADS), VARMUL_COMB_THREADS, COMB_BASE_DOUBLES * sizeof(double), st>>>(
            (const uint32_t *)s, s_step, pl.table, m, pl.clamp, (uint32_t *)out, (uint8_t *)ok, pl.status);
    else
        k_varmul<FMT><<<cdiv(m, VARMUL_THREADS), VARMUL_THREADS, 0, st>>>((const uint32_t *)s, s_step, (const uint32_t *)p, p_step, m,
                                                                          pl.clamp, (uint32_t *)out, (uint8_t *)ok, pl.status);
}

static void varmul_launch(const VarmulPlan &pl, const void *s, size_t s_step, const void *p, size_t p_step, size_t m, void *out, void *ok,
                          cudaStream_t st)
{
    if (pl.fmt == DALEK_POINTS_EXTENDED) varmul_launch_fmt<DALEK_POINTS_EXTENDED>(pl, s, s_step, p, p_step, m, out, ok, st);
    else if (pl.fmt == DALEK_POINTS_RISTRETTO) varmul_launch_fmt<DALEK_POINTS_RISTRETTO>(pl, s, s_step, p, p_step, m, out, ok, st);
    else varmul_launch_fmt<DALEK_POINTS_COMPRESSED>(pl, s, s_step, p, p_step, m, out, ok, st);
}

template <int FMT>
static int varmul_comb_table_fmt(dalek_b200_ctx *ctx, const void *d_point, double *table, int *status)
{
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_varmul_comb<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(COMB_BASE_DOUBLES * sizeof(double))));
    k_varmul_comb_table<FMT><<<4, 128, 0, ctx->stream>>>((const uint32_t *)d_point, table, status);
    return 0;
}

// argument checks shared by both calls, and the choice of path
static int varmul_setup(dalek_b200_ctx *ctx, size_t n_scalars, int point_fmt, size_t n_points, size_t n, int flags, VarmulPlan &pl)
{
    if ((n_scalars != 1 && n_scalars != n) || (n_points != 1 && n_points != n)) {
        ctx->last_error = "n_scalars and n_points must each be 1 or n";
        return DALEK_E_INVALID_ARG;
    }
    if (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED && point_fmt != DALEK_POINTS_RISTRETTO) return DALEK_E_INVALID_ARG;
    if (flags & ~DALEK_MUL_CLAMPED) return DALEK_E_INVALID_ARG;
    if ((flags & DALEK_MUL_CLAMPED) && point_fmt == DALEK_POINTS_RISTRETTO) {
        ctx->last_error = "clamped multiplication is defined for Edwards points only";
        return DALEK_E_INVALID_ARG;
    }
    pl.fmt = point_fmt;
    pl.clamp = (flags & DALEK_MUL_CLAMPED) ? 1u : 0u;
    pl.comb = n_points == 1 && n >= VARMUL_COMB_MIN;
    return 0;
}

// the status word cleared and, for the comb path, the table of the point at d_point (device) enqueued on ctx->stream
static int varmul_prepare(dalek_b200_ctx *ctx, VarmulPlan &pl, const void *d_point)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_TABLE + COMB_BASE_DOUBLES * sizeof(double)))) return rc;
    char *base = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    pl.status = (int *)(base + VM_STATUS);
    pl.table = (const double *)(base + VM_TABLE);
    CUDA_TRY(ctx, cudaMemsetAsync(pl.status, 0, 4, ctx->stream));
    if (pl.comb) {
        if (pl.fmt == DALEK_POINTS_EXTENDED) rc = varmul_comb_table_fmt<DALEK_POINTS_EXTENDED>(ctx, d_point, (double *)pl.table, pl.status);
        else if (pl.fmt == DALEK_POINTS_RISTRETTO) rc = varmul_comb_table_fmt<DALEK_POINTS_RISTRETTO>(ctx, d_point, (double *)pl.table, pl.status);
        else rc = varmul_comb_table_fmt<DALEK_POINTS_COMPRESSED>(ctx, d_point, (double *)pl.table, pl.status);
        if (rc) return rc;
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return 0;
}

static int varmul_read_status(dalek_b200_ctx *ctx, const int *d_status, int *status)
{
    int rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *status = *(const int *)ctx->h_pinned;
    return 0;
}

template <int FMT>
static void torsion_launch_fmt(const void *p, size_t m, void *out, cudaStream_t st)
{
    k_torsion<FMT><<<cdiv(m, VARMUL_THREADS), VARMUL_THREADS, 0, st>>>((const uint32_t *)p, m, (uint8_t *)out);
}

extern "C" {

int dalek_b200_mul_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n_scalars, const void *points, int point_fmt,
                         size_t n_points, size_t n, int flags, uint8_t *out, uint8_t *ok)
{
    if (!ctx || (n && (!scalars || !points || !out))) return DALEK_E_INVALID_ARG;
    VarmulPlan pl;
    int rc;
    if ((rc = varmul_setup(ctx, n_scalars, point_fmt, n_points, n, flags, pl))) return rc;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    if (!pl.clamp) {                                               // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear
        uint8_t top = 0;
        for (size_t i = 0; i < n_scalars; i++) top |= scalars[32 * i + 31];
        if (top & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    }
    CallTimer timer(ctx);
    const size_t pin = msm_point_bytes(point_fmt);
    const bool bs = n_scalars == 1, bp = n_points == 1;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_TABLE + COMB_BASE_DOUBLES * sizeof(double)))) return rc;
    char *base = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    if (bs) CUDA_TRY(ctx, cudaMemcpyAsync(base + VM_SCALAR, scalars, 32, cudaMemcpyHostToDevice, ctx->stream));
    if (bp) CUDA_TRY(ctx, cudaMemcpyAsync(base + VM_POINT, points, pin, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = varmul_prepare(ctx, pl, base + VM_POINT))) return rc;
    const size_t s_sz = bs ? 0 : 32, p_sz = bp ? 0 : pin, ok_sz = ok ? 1 : 0;
    rc = run_pieces(ctx, nullptr, nullptr, bs ? nullptr : scalars, s_sz, bp ? nullptr : (const uint8_t *)points, p_sz, out, 32, ok, ok_sz, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_s, const uint8_t *d_p, size_t m, uint8_t *d_o, uint8_t *d_ok,
                        cudaStream_t st) {
                        varmul_launch(pl, bs ? base + VM_SCALAR : (const char *)d_s, bs ? 0 : 1, bp ? base + VM_POINT : (const char *)d_p,
                                      bp ? 0 : 1, m, d_o, ok ? d_ok : nullptr, st);
                        return 0;
                    });
    if (rc) return rc;
    int status = 0;
    if ((rc = varmul_read_status(ctx, pl.status, &status))) return rc;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_IN].p, 0, std::max<size_t>(1, n) * (s_sz + p_sz), ctx->stream));   // zeroize on drop
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_OUT].p, 0, std::max<size_t>(1, n) * (32 + ok_sz), ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(base + VM_SCALAR, 0, 32, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return (status & VM_BAD_POINT) ? DALEK_NONE : DALEK_OK;
}

int dalek_b200_mul_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, size_t n_scalars, const void *d_points, int point_fmt,
                             size_t n_points, size_t n, int flags, void *d_out, void *d_ok)
{
    if (!ctx || (n && (!d_scalars || !d_points || !d_out))) return DALEK_E_INVALID_ARG;
    VarmulPlan pl;
    int rc;
    if ((rc = varmul_setup(ctx, n_scalars, point_fmt, n_points, n, flags, pl))) return rc;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    if ((rc = varmul_prepare(ctx, pl, d_points))) return rc;
    varmul_launch(pl, d_scalars, n_scalars == 1 ? 0 : 1, d_points, n_points == 1 ? 0 : 1, n, d_out, d_ok,
                  ctx->stream);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    int status = 0;
    if ((rc = varmul_read_status(ctx, pl.status, &status))) return rc;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = pl.comb ? 2 : 1;
    if (status & VM_BAD_SCALAR) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    return (status & VM_BAD_POINT) ? DALEK_NONE : DALEK_OK;
}

int dalek_b200_edwards_torsion_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!points || !out))) return DALEK_E_INVALID_ARG;
    if (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_pieces(ctx, nullptr, nullptr, (const uint8_t *)points, msm_point_bytes(point_fmt), nullptr, 0, out, 1, nullptr, 0, n,
                      [&](const uint8_t *, const uint64_t *, const uint8_t *d_p, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                          cudaStream_t st) {
                          if (point_fmt == DALEK_POINTS_EXTENDED) torsion_launch_fmt<DALEK_POINTS_EXTENDED>(d_p, m, d_o, st);
                          else torsion_launch_fmt<DALEK_POINTS_COMPRESSED>(d_p, m, d_o, st);
                          return 0;
                      });
}

}  // extern "C"
