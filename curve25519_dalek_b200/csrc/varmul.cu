// varmul.cu -- batched variable-base scalar multiplication out[i] = s_i P_i, resident basepoint tables, and the torsion
// checks of Edwards points.
//   EdwardsPoint * Scalar           C/edwards.rs:890-899 -> variable_base.rs:11-48   k_varmul       one thread per item
//   EdwardsPoint::mul_clamped       C/edwards.rs:932-941                               (clamped, not reduced)
//   RistrettoPoint * Scalar         C/ristretto.rs:917-926
//   BasepointTable::create(P)       C/traits.rs:50-74, C/edwards.rs:1127-1243,          k_comb_pow16 + k_comb_rows
//     basepoint, mul_base,          C/ristretto.rs:1080-1115                           k_varmul_comb (one table),
//     mul_base_clamped                                                                 k_bpt_mul (many tables)
//   is_small_order / is_torsion_free C/edwards.rs:1405-1437                           k_torsion
// k_varmul decodes P_i, runs varmul.cuh on the FP64 field with its [P..8P] table in local memory, and encodes the
// result.  When one point serves a batch of at least VARMUL_COMB_MIN items, its 64 x 8 comb table (comb.cuh) is built
// once per call and every item costs 64 mixed additions and no doubling; both paths give the same bytes.  A basepoint
// table handle keeps the comb tables of k points resident in device memory, built by the same two kernels.
// Constant time in the scalars: no branch, loop bound or address depends on them (varmul.cuh; comb.cuh scans every
// entry of a table row).  The one exception is the report of a scalar with bit 255 set by a device-buffer call, which
// fails the call.  Points and table indices are public.  Host-buffer calls clear the device copies of the scalars and
// of the results before they return.
#include <algorithm>
#include <cstring>
#include <new>

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
#define BPT_THREADS 128               // k_bpt_mul
#define BPT_BUILD_GROUP 4096          // points per pass of a table build: their 16^i P take 40 MiB

// staging in WS_CALL_SCRATCH: status word, the broadcast scalar, the broadcast point, the comb table, the 16^i P of its build
#define VM_STATUS 0
#define VM_SCALAR 64
#define VM_POINT 128
#define VM_TABLE 512
#define VM_POW (VM_TABLE + COMB_BASE_DOUBLES * 8)
#define VM_END (VM_POW + 64 * sizeof(ge_p3_raw))

enum { VM_BAD_POINT = 1, VM_BAD_SCALAR = 2, VM_BAD_INDEX = 4 };

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

// ---- comb tables of k points: entry j of row i of table p = (j+1) 16^i P_p (comb.cuh layout, COMB_BASE_DOUBLES each) --
// one thread per point: decode P_p, then 16^i P_p for i = 0..63 (63 x 4 doublings, shared by the table's 512 entries)
template <int FMT>
__global__ void __launch_bounds__(64)
k_comb_pow16(const uint32_t *__restrict__ points, size_t k, ge_p3_raw *__restrict__ pw, uint8_t *__restrict__ ok, int *status)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= k) return;
    ge_p3 A;
    const uint32_t good = varmul_load_point<FMT>(A, points, p);
    if (ok) ok[p] = (uint8_t)good;
    if (!good) atomicOr(status, VM_BAD_POINT);                     // the points are public
    ge64_p3 P; ge64_from_p3(P, A);
#pragma unroll 1
    for (int pos = 0; pos < 64; pos++) {
        if (pos) { ge64_dbl(P, P); ge64_dbl(P, P); ge64_dbl(P, P); ge64_dbl(P, P); }
        ge_p3 q; ge64_to_p3(q, P);
        ge_p3_raw r; ge_p3_store_raw(r, q);
        uint4 *o = reinterpret_cast<uint4 *>(pw + p * 64 + pos);
#pragma unroll
        for (int w = 0; w < 10; w++) o[w] = make_uint4(r.w[4 * w], r.w[4 * w + 1], r.w[4 * w + 2], r.w[4 * w + 3]);
    }
}

// one thread per table entry: (j+1) 16^i P_p from 16^i P_p with j additions and one inversion, as affine Niels
// coordinates in balanced FP64 limbs
__global__ void __launch_bounds__(128)
k_comb_rows(const ge_p3_raw *__restrict__ pw, size_t k, double *__restrict__ tab)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k * 512) return;
    const int j = (int)(t & 7);
    ge_p3 P;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(pw + (t >> 3));
        ge_p3_raw r;
#pragma unroll
        for (int w = 0; w < 10; w++) { uint4 v = src[w]; r.w[4 * w] = v.x; r.w[4 * w + 1] = v.y; r.w[4 * w + 2] = v.z; r.w[4 * w + 3] = v.w; }
        ge_p3_load_raw(P, r);
    }
    ge_pniels nb; ge_p3_to_pniels(nb, P);
    ge_p3 Q = P;
#pragma unroll 1
    for (int m = 0; m < j; m++) ge_padd(Q, Q, nb, 0);
    fe zi, x, y;
    fe_invert_f64(zi, Q.Z);
    fe_mul(x, Q.X, zi); fe_mul(y, Q.Y, zi);
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    fe64 e[3];
    fe64_from_fe(e[0], nl.ypx); fe64_from_fe(e[1], nl.ymx); fe64_from_fe(e[2], nl.xy2d);
    double *dst = tab + t * COMB_ENTRY;
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int m = 0; m < 5; m++) dst[5 * c + m] = e[c].v[m];
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

// out[i] = s_i P_{t_i} from table t_i of the k tables in global memory, every row scanned in full.  Thread j takes item
// order[j] (order NULL: item j), so that with the items grouped by table the lanes of a warp read the same rows.  The
// index is public; one >= k reads table 0 and fails the call.
template <int FMT>
__global__ void __launch_bounds__(BPT_THREADS)
k_bpt_mul(const uint32_t *__restrict__ scalars, const uint32_t *__restrict__ indices, const uint32_t *__restrict__ order, size_t n,
          const double *__restrict__ tables, size_t k, uint32_t clamp, uint32_t *__restrict__ out, int *status)
{
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const size_t i = order ? order[j] : j;
    uint32_t s[8];
    varmul_load_scalar(s, scalars, 1, i, clamp, status);
    const uint32_t t = indices[i];
    const bool bad = t >= k;
    if (bad) atomicOr(status, VM_BAD_INDEX);
    ge64_p3 Q;
    comb_mul_base(Q, s, tables + (size_t)(bad ? 0u : t) * COMB_BASE_DOUBLES);
    varmul_encode<FMT>(out + 8 * i, Q);
}

// ---- the items of a many-table call grouped by table: a counting sort of the (public) indices -------------------------
// cnt[t] = the number of items of table t (an index >= k counts as 0; k_bpt_mul fails the call for it)
__global__ void __launch_bounds__(256) k_bpt_count(const uint32_t *__restrict__ indices, size_t n, size_t k, uint32_t *__restrict__ cnt)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t t = indices[i];
    atomicAdd(&cnt[t < k ? t : 0u], 1u);
}

// cnt[0..k) -> its exclusive prefix sums, in place: one block, each thread a run of consecutive tables
__global__ void __launch_bounds__(1024) k_bpt_offsets(uint32_t *__restrict__ cnt, size_t k)
{
    __shared__ uint32_t part[1024];
    const size_t per = (k + 1023) / 1024, a = threadIdx.x * per, lo = a < k ? a : k, hi = lo + per < k ? lo + per : k;
    uint32_t sum = 0;
    for (size_t t = lo; t < hi; t++) sum += cnt[t];
    part[threadIdx.x] = sum;
    __syncthreads();
    for (unsigned off = 1; off < 1024; off <<= 1) {
        const uint32_t v = threadIdx.x >= off ? part[threadIdx.x - off] : 0u;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - sum;
    for (size_t t = lo; t < hi; t++) { const uint32_t c = cnt[t]; cnt[t] = run; run += c; }
}

// order[offset of t_i + rank] = i: the items of each table together (their order inside a table is immaterial)
__global__ void __launch_bounds__(256)
k_bpt_order(const uint32_t *__restrict__ indices, size_t n, size_t k, uint32_t *__restrict__ cnt, uint32_t *__restrict__ order)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t t = indices[i];
    order[atomicAdd(&cnt[t < k ? t : 0u], 1u)] = (uint32_t)i;
}

// the indices of a device-buffer call served by its one table are all 0
__global__ void __launch_bounds__(128) k_bpt_check_indices(const uint32_t *__restrict__ indices, size_t n, int *status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && indices[i] != 0) atomicOr(status, VM_BAD_INDEX);
}

// out[p] = the encoding of P_p, read back from entry (0, 0) = (y + x, y - x, 2dxy) of table p (C/edwards.rs:1144-1148)
template <int FMT>
__global__ void __launch_bounds__(128) k_bpt_basepoints(const double *__restrict__ tables, size_t k, uint32_t *__restrict__ out)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= k) return;
    const double *e = tables + p * COMB_BASE_DOUBLES;
    fe64 a, b;
#pragma unroll
    for (int m = 0; m < 5; m++) { a.v[m] = e[m]; b.v[m] = e[5 + m]; }
    fe ypx, ymx, half, t;
    fe64_to_fe(ypx, a); fe64_to_fe(ymx, b);
    const uint32_t half_words[8] = {0xfffffff7u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
    fe_frombytes_words(half, half_words);                         // (p + 1) / 2 = 2^254 - 9
    ge_p3 P;
    fe_sub(t, ypx, ymx); fe_mul(P.X, t, half);
    fe_add(t, ypx, ymx); fe_mul(P.Y, t, half);
    fe_1(P.Z);
    fe_mul(P.T, P.X, P.Y);
    uint32_t w[8];
    if (FMT == DALEK_POINTS_RISTRETTO) ristretto_compress<1>(w, P);
    else ge_compress<1>(w, P);
#pragma unroll
    for (int m = 0; m < 8; m++) out[8 * p + m] = w[m];
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
static int varmul_comb_smem_fmt(dalek_b200_ctx *ctx)
{
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_varmul_comb<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(COMB_BASE_DOUBLES * sizeof(double))));
    return 0;
}

// k_varmul_comb's table is staged in dynamic shared memory
static int varmul_comb_smem(dalek_b200_ctx *ctx, int fmt)
{
    if (fmt == DALEK_POINTS_EXTENDED) return varmul_comb_smem_fmt<DALEK_POINTS_EXTENDED>(ctx);
    if (fmt == DALEK_POINTS_RISTRETTO) return varmul_comb_smem_fmt<DALEK_POINTS_RISTRETTO>(ctx);
    return varmul_comb_smem_fmt<DALEK_POINTS_COMPRESSED>(ctx);
}

// the comb tables of the k points at d_points (device, format fmt) into `tables` (k x COMB_BASE_DOUBLES), enqueued on
// ctx->stream in passes of `group` points whose 16^i P go to pw (group x 64).  An undecodable point gets the identity's
// table, ok[p] = 0 (d_ok device, nullable) and VM_BAD_POINT in *status.
static int comb_tables_build(dalek_b200_ctx *ctx, int fmt, const void *d_points, size_t k, ge_p3_raw *pw, size_t group,
                             double *tables, uint8_t *d_ok, int *status)
{
    const size_t pin = msm_point_bytes(fmt);
    cudaStream_t st = ctx->stream;
    for (size_t lo = 0; lo < k; lo += group) {
        const size_t g = std::min(group, k - lo);
        const uint32_t *pts = (const uint32_t *)((const char *)d_points + lo * pin);
        uint8_t *ok = d_ok ? d_ok + lo : nullptr;
        if (fmt == DALEK_POINTS_EXTENDED) k_comb_pow16<DALEK_POINTS_EXTENDED><<<cdiv(g, 64), 64, 0, st>>>(pts, g, pw, ok, status);
        else if (fmt == DALEK_POINTS_RISTRETTO) k_comb_pow16<DALEK_POINTS_RISTRETTO><<<cdiv(g, 64), 64, 0, st>>>(pts, g, pw, ok, status);
        else k_comb_pow16<DALEK_POINTS_COMPRESSED><<<cdiv(g, 64), 64, 0, st>>>(pts, g, pw, ok, status);
        k_comb_rows<<<cdiv(g * 512, 128), 128, 0, st>>>(pw, g, tables + lo * COMB_BASE_DOUBLES);
        ctx->launches += 2;
        CUDA_TRY(ctx, cudaGetLastError());
    }
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
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_END))) return rc;
    char *base = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    pl.status = (int *)(base + VM_STATUS);
    pl.table = (const double *)(base + VM_TABLE);
    CUDA_TRY(ctx, cudaMemsetAsync(pl.status, 0, 4, ctx->stream));
    if (pl.comb) {
        if ((rc = varmul_comb_smem(ctx, pl.fmt))) return rc;
        if ((rc = comb_tables_build(ctx, pl.fmt, d_point, 1, (ge_p3_raw *)(base + VM_POW), 1, (double *)pl.table, nullptr, pl.status)))
            return rc;
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

// ---- resident basepoint tables ----------------------------------------------------------------------------------------
struct dalek_b200_basepoint_tables {
    dalek_b200_ctx *ctx;   // the context it serves; destroy does not touch it
    int device;
    double *d_tables;      // k x COMB_BASE_DOUBLES, device
    size_t k;
    int fmt;               // DALEK_POINTS_COMPRESSED (Edwards tables) or DALEK_POINTS_RISTRETTO (Ristretto tables)
};

// argument checks shared by the two multiplication calls
static int bpt_check(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, const void *scalars, size_t n, int flags,
                     const void *out)
{
    if (!ctx || !t || (n && (!scalars || !out)) || (flags & ~DALEK_MUL_CLAMPED)) return DALEK_E_INVALID_ARG;
    if (t->ctx != ctx) { ctx->last_error = "basepoint tables used with a context other than their own"; return DALEK_E_INVALID_ARG; }
    return 0;
}

// the status word cleared and, for the one-table path, k_varmul_comb's shared-memory limit set
static int bpt_prepare(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, bool one, int **status)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_END))) return rc;
    *status = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + VM_STATUS);
    CUDA_TRY(ctx, cudaMemsetAsync(*status, 0, 4, ctx->stream));
    if (one && (rc = varmul_comb_smem(ctx, t->fmt))) return rc;
    return 0;
}

// the workspace of the grouping: a table count array per stream, then one order entry per item
static int bpt_order_reserve(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, size_t n)
{
    return ws_reserve(ctx, ctx->ws[WS_BPT_ORDER], (2 * t->k + n) * sizeof(uint32_t));
}

// enqueue the order of the m items at idx (piece starting at item lo) grouped by table into *order; NULL when the
// context does not group (option "bpt_group" 0)
static int bpt_group(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, const void *idx, size_t m, size_t lo, cudaStream_t st,
                     const uint32_t **order)
{
    *order = nullptr;
    if (!ctx->opt_bpt_group) return 0;
    uint32_t *cnt = (uint32_t *)ctx->ws[WS_BPT_ORDER].p + (st == ctx->stream ? 0 : t->k);
    uint32_t *ord = (uint32_t *)ctx->ws[WS_BPT_ORDER].p + 2 * t->k + lo;
    CUDA_TRY(ctx, cudaMemsetAsync(cnt, 0, t->k * sizeof(uint32_t), st));
    k_bpt_count<<<cdiv(m, 256), 256, 0, st>>>((const uint32_t *)idx, m, t->k, cnt);
    k_bpt_offsets<<<1, 1024, 0, st>>>(cnt, t->k);
    k_bpt_order<<<cdiv(m, 256), 256, 0, st>>>((const uint32_t *)idx, m, t->k, cnt, ord);
    ctx->launches += 3;
    *order = ord;
    return 0;
}

// one launch of m items: through table 0 (one), or through table indices[i] of each item in the given order
template <int FMT>
static void bpt_launch_fmt(const dalek_b200_basepoint_tables *t, bool one, const void *s, const void *idx, const uint32_t *order, size_t m,
                           uint32_t clamp, void *out, int *status, cudaStream_t st)
{
    if (one)
        k_varmul_comb<FMT><<<cdiv(m, VARMUL_COMB_THREADS), VARMUL_COMB_THREADS, COMB_BASE_DOUBLES * sizeof(double), st>>>(
            (const uint32_t *)s, 1, t->d_tables, m, clamp, (uint32_t *)out, nullptr, status);
    else
        k_bpt_mul<FMT><<<cdiv(m, BPT_THREADS), BPT_THREADS, 0, st>>>((const uint32_t *)s, (const uint32_t *)idx, order, m, t->d_tables,
                                                                     t->k, clamp, (uint32_t *)out, status);
}

static int bpt_launch(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, bool one, const void *s, const void *idx, size_t m,
                      size_t lo, uint32_t clamp, void *out, int *status, cudaStream_t st)
{
    const uint32_t *order = nullptr;
    int rc;
    if (!one && (rc = bpt_group(ctx, t, idx, m, lo, st, &order))) return rc;
    if (t->fmt == DALEK_POINTS_RISTRETTO) bpt_launch_fmt<DALEK_POINTS_RISTRETTO>(t, one, s, idx, order, m, clamp, out, status, st);
    else bpt_launch_fmt<DALEK_POINTS_COMPRESSED>(t, one, s, idx, order, m, clamp, out, status, st);
    return 0;
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
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_END))) return rc;
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
    ctx->last_kernel_launches = pl.comb ? 3 : 1;
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

int dalek_b200_basepoint_tables_new(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t k, uint8_t *ok,
                                    dalek_b200_basepoint_tables **out)
{
    if (!ctx || !out) return DALEK_E_INVALID_ARG;
    *out = nullptr;
    if (!points || !k || k > 0xffffffffull) return DALEK_E_INVALID_ARG;
    if (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED && point_fmt != DALEK_POINTS_RISTRETTO)
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    const size_t pin = msm_point_bytes(point_fmt), group = std::min<size_t>(k, BPT_BUILD_GROUP);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], k * pin))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], k))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], VM_END))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    dalek_b200_basepoint_tables *t = new (std::nothrow) dalek_b200_basepoint_tables();
    if (!t) { ctx->last_error = "out of host memory for the basepoint tables"; return DALEK_E_NOMEM; }
    t->ctx = ctx; t->device = ctx->device; t->k = k; t->fmt = point_fmt == DALEK_POINTS_RISTRETTO ? DALEK_POINTS_RISTRETTO : DALEK_POINTS_COMPRESSED;
    t->d_tables = nullptr;
    ge_p3_raw *pw = nullptr;
    auto fail = [&](int code) {
        cudaFree(pw); cudaFree(t->d_tables); delete t;
        return code;
    };
    if (cudaMalloc((void **)&t->d_tables, k * COMB_BASE_DOUBLES * sizeof(double)) != cudaSuccess ||
        cudaMalloc((void **)&pw, group * 64 * sizeof(ge_p3_raw)) != cudaSuccess) {
        (void)cudaGetLastError();
        ctx->last_error = "cudaMalloc failed for the basepoint tables";
        return fail(DALEK_E_NOMEM);
    }
    auto cuda_fail = [&]() {
        ctx->last_error = std::string("basepoint table build: ") + cudaGetErrorString(cudaGetLastError());
        return fail(DALEK_E_CUDA);
    };
    int *status = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + VM_STATUS);
    uint8_t *d_ok = (uint8_t *)ctx->ws[WS_STAGING_OUT].p;
    cudaStream_t st = ctx->stream;
    if (cudaEventRecord(ctx->ev_a, st) != cudaSuccess || cudaMemsetAsync(status, 0, 4, st) != cudaSuccess ||
        cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, points, k * pin, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cuda_fail();
    if ((rc = comb_tables_build(ctx, point_fmt, ctx->ws[WS_STAGING_IN].p, k, pw, group, t->d_tables, d_ok, status))) return fail(rc);
    if ((ok && cudaMemcpyAsync(ok, d_ok, k, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaMemcpyAsync(ctx->h_pinned, status, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaEventRecord(ctx->ev_b, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cuda_fail();
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)(2 * ((k + group - 1) / group));
    cudaFree(pw); pw = nullptr;
    if (*(const int *)ctx->h_pinned & VM_BAD_POINT) { ctx->last_error = "a point does not decode"; return fail(DALEK_NONE); }
    *out = t;
    return DALEK_OK;
}

size_t dalek_b200_basepoint_tables_len(const dalek_b200_basepoint_tables *t) { return t ? t->k : 0; }

void dalek_b200_basepoint_tables_destroy(dalek_b200_basepoint_tables *t)
{
    if (!t) return;
    cudaSetDevice(t->device);
    cudaFree(t->d_tables);                                         // waits for the device: no call still reads the tables
    delete t;
}

int dalek_b200_basepoint_tables_basepoints(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, uint8_t *out)
{
    if (!ctx || !t || !out) return DALEK_E_INVALID_ARG;
    if (t->ctx != ctx) { ctx->last_error = "basepoint tables used with a context other than their own"; return DALEK_E_INVALID_ARG; }
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], t->k * 32))) return rc;
    uint32_t *d_out = (uint32_t *)ctx->ws[WS_STAGING_OUT].p;
    if (t->fmt == DALEK_POINTS_RISTRETTO)
        k_bpt_basepoints<DALEK_POINTS_RISTRETTO><<<cdiv(t->k, 128), 128, 0, ctx->stream>>>(t->d_tables, t->k, d_out);
    else
        k_bpt_basepoints<DALEK_POINTS_COMPRESSED><<<cdiv(t->k, 128), 128, 0, ctx->stream>>>(t->d_tables, t->k, d_out);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(out, d_out, t->k * 32, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return DALEK_OK;
}

int dalek_b200_basepoint_tables_mul(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, const uint8_t *scalars,
                                    const uint32_t *indices, size_t n, int flags, uint8_t *out)
{
    int rc;
    if ((rc = bpt_check(ctx, t, scalars, n, flags, out))) return rc;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    const uint32_t clamp = (flags & DALEK_MUL_CLAMPED) ? 1u : 0u;
    if (!clamp) {                                                  // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear
        uint8_t top = 0;
        for (size_t i = 0; i < n; i++) top |= scalars[32 * i + 31];
        if (top & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    }
    if (indices)                                                   // public: checked before any device work
        for (size_t i = 0; i < n; i++)
            if (indices[i] >= t->k) { ctx->last_error = "table index >= len()"; return DALEK_E_INVALID_ARG; }
    CallTimer timer(ctx);
    const bool one = !indices || t->k == 1;
    int *status = nullptr;
    if ((rc = bpt_prepare(ctx, t, one, &status))) return rc;
    const size_t i_sz = one ? 0 : 4;
    if (!one && (rc = bpt_order_reserve(ctx, t, n))) return rc;
    rc = run_pieces(ctx, nullptr, nullptr, scalars, 32, one ? nullptr : (const uint8_t *)indices, i_sz, out, 32, nullptr, 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_s, const uint8_t *d_i, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st, size_t lo) {
                        return bpt_launch(ctx, t, one, d_s, d_i, m, lo, clamp, d_o, status, st);
                    });
    // zeroize on drop, failed calls included: the staged scalars and results, as far as they were reserved
    const size_t in_b = std::min(n * (32 + i_sz), ctx->ws[WS_STAGING_IN].cap), out_b = std::min(n * 32, ctx->ws[WS_STAGING_OUT].cap);
    const int wipe = wipe_staging(ctx, in_b, out_b);
    return rc ? rc : wipe;
}

int dalek_b200_basepoint_tables_mul_dev(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t, const void *d_scalars,
                                        const void *d_indices, size_t n, int flags, void *d_out)
{
    int rc;
    if ((rc = bpt_check(ctx, t, d_scalars, n, flags, d_out))) return rc;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const uint32_t clamp = (flags & DALEK_MUL_CLAMPED) ? 1u : 0u;
    const bool one = !d_indices || t->k == 1;
    int *status = nullptr;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    if ((rc = bpt_prepare(ctx, t, one, &status))) return rc;
    int launches = 1;
    if (one && d_indices) {
        k_bpt_check_indices<<<cdiv(n, 128), 128, 0, ctx->stream>>>((const uint32_t *)d_indices, n, status);
        ctx->launches++;
        launches++;
    }
    if (!one) {
        if ((rc = bpt_order_reserve(ctx, t, n))) return rc;
        launches += ctx->opt_bpt_group ? 3 : 0;
    }
    if ((rc = bpt_launch(ctx, t, one, d_scalars, d_indices, n, 0, clamp, d_out, status, ctx->stream))) return rc;
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    int st = 0;
    if ((rc = varmul_read_status(ctx, status, &st))) return rc;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = launches;
    if (st & VM_BAD_SCALAR) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    if (st & VM_BAD_INDEX) { ctx->last_error = "table index >= len()"; return DALEK_E_INVALID_ARG; }
    return DALEK_OK;
}

}  // extern "C"
