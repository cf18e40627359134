// msm.cu -- bucket-method (Pippenger) multiscalar multiplication on one H100.
//
// Replaces curve25519-dalek/src/backend/serial/scalar_mul/pippenger.rs:67-160 (and, being
// size-agnostic, the vartime Straus path straus.rs:159-200 the reference dispatches to below 190
// points, src/edwards.rs:1025-1029).  The reference walks 33-43 windows of 6-8 bits serially;
// here all windows run at once with c = 4..20-bit signed digits:
//
//   k_sort_count/bins_scan/partition/fine
//                       signed radix-2^c digits (scalar.rs:1093-1150 generalised to c > 8), point indices
//                       grouped by (window, bucket) in a two-level counting sort: coarse bins of 2^F buckets
//                       through HBM, the low F bits in shared memory; bucket sizes and offsets
//   k_task_count, k_scan_*
//                       buckets cut into tasks of <= task_len entries (skewed / adversarial inputs), per-window
//                       exclusive scan of the task counts (multi-block)
//   k_task_fill
//   k_task_hist/scan/scatter
//                       counting sort of the tasks by length: warps run equal trip counts and the
//                       grid drains longest-first
//   k_bucket_accumulate one thread per task: sum of its points with the complete unified mixed
//                       addition of an affine Niels point (curve_models.rs:411-494), 7M, on the
//                       FP64-pipe field (fe64.cuh) with cp.async point prefetch
//   k_heavy_fixup       sums the task sums of buckets that were cut
//   k_chunk_reduce, k_plain_sum, k_finish_windows
//                       sum_k k*B_k per window (pippenger.rs:146-151) in log depth on 4-lane groups
//   k_combine           total = total*2^c + window (pippenger.rs:159), compress
//
// Data layout in HBM: scalars n x 32 B; points packed affine Niels (96 B: every input format is normalised
// to Z = 1 first), canonical 32-byte coordinates, 16-byte aligned for 128-bit loads; sort records 8 B per
// non-zero digit; sorted indices 4 B per entry; bucket sums 160 B (10 x u32 limbs x 4).
#include <algorithm>
#include <cstdio>
#include <utility>
#include <vector>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "ge64.cuh"
#include "warp4.cuh"
#include "warp4_f64.cuh"

// ------------------------------------------------------------------------------------------
static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

int ws_reserve(dalek_b200_ctx *ctx, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return 0;
    if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
        ctx->last_error = std::string("cudaMalloc: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();        // else the next CUDA_TRY(cudaGetLastError()) of this host thread reports it
        return DALEK_E_NOMEM;
    }
    b.cap = want;
    return 0;
}

int pinned_reserve(dalek_b200_ctx *ctx, size_t bytes)
{
    if (bytes <= ctx->h_pinned_cap) return 0;
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    ctx->h_pinned = nullptr; ctx->h_pinned_cap = 0;
    cudaError_t e = cudaMallocHost(&ctx->h_pinned, bytes + 4096);
    if (e != cudaSuccess) {
        ctx->last_error = std::string("cudaMallocHost: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();
        return DALEK_E_NOMEM;
    }
    ctx->h_pinned_cap = bytes + 4096;
    return 0;
}

// ------------------------------------------------------------------------------------------
// point preparation
template <int F64>
__global__ void __launch_bounds__(128, 3) k_prep_compressed(const uint4 *__restrict__ in, ge_niels_packed *__restrict__ out, size_t n,
                                  int *__restrict__ bad)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint4 a = in[2 * i], b = in[2 * i + 1];
    uint32_t s[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    fe x, y;
    uint32_t ok = ge_decompress_affine<F64>(x, y, s);
    if (!ok) { atomicOr(bad, 1); fe_0(x); fe_1(y); }   // identity placeholder keeps the kernels total
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    ge_niels_packed p; ge_niels_pack(p, nl);
    uint4 *o = reinterpret_cast<uint4 *>(out + i);
#pragma unroll
    for (int k = 0; k < 6; k++) o[k] = make_uint4(p.w[4 * k], p.w[4 * k + 1], p.w[4 * k + 2], p.w[4 * k + 3]);
}

// CompressedRistretto -> affine Niels with the Ristretto decoding rules (ristretto.rs:266-345); the decoded point is
// affine (Z = 1), so it goes straight to the form of the bucket kernel
template <int F64>
__global__ void k_prep_ristretto(const uint32_t *__restrict__ in, ge_niels_packed *__restrict__ out, size_t n, int *__restrict__ bad)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t enc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) enc[k] = in[8 * i + k];
    ge_p3 P;
    if (!ristretto_decompress<F64>(P, enc)) { atomicOr(bad, 1); ge_p3_identity(P); }
    ge_niels nl; ge_affine_to_niels(nl, P.X, P.Y);
    ge_niels_packed pk; ge_niels_pack(pk, nl);
    out[i] = pk;
}

// Extended points (X : Y : Z : T) -> affine Niels ((Y+X)/Z, (Y-X)/Z, 2d T/Z): the projective Niels point divided by Z,
// so every input with Z != 0 stands for the same group element as before, T/Z = xy or not.  The bucket kernel then
// adds every point with the 7M mixed addition in each of its ~16 windows instead of the 8M projective one, and
// gathers 96 B per digit instead of 128 B.  All the inversions are one Montgomery batch over the whole input, in three
// short grid-wide passes over groups of PREP_GROUP points (one CTA per group):
//   k_prep_zprod   the product of the Z of each group
//   k_prep_invert  one CTA: the inverses of all the group products, with one field inversion
//   k_prep_finish  each group again: the product of each thread's Z, its inverse from the group's inverse (Montgomery's
//                  trick across the CTA), then every thread walks its points backwards and writes them
// No CTA of the first and last pass waits on a serial inversion, so their CTAs are short and the digit sort of the main
// stream gets SMs soon after it asks for them.  Z = 0 (not a point: bad limbs from the caller) is left out of the
// products, as FieldElement::invert_batch skips zeros, and gives the identity; the other points of its group are
// unaffected.
#define PREP_THREADS 256
#define PREP_PER_THREAD 4
#define PREP_GROUP (PREP_THREADS * PREP_PER_THREAD)      // points per group: point k of thread t is base + k * PREP_THREADS + t
#define PREP_NW (PREP_THREADS / 32)

__device__ __forceinline__ void load_coord_f64(fe64 &h, const uint64_t *__restrict__ src)
{
    uint64_t l[5];
#pragma unroll
    for (int k = 0; k < 5; k++) l[k] = __ldg(src + k);
    fe t; fe_from_limbs51(t, l);
    fe64_from_fe_limbs(h, t);
}
// the canonical 32 bytes of v if ok, else of the small constant c, to o[0], o[1]
__device__ __forceinline__ void store_coord(uint4 *o, const fe64 &v, uint32_t ok, uint32_t c)
{
    fe f;
    uint32_t w[8];
    fe64_to_fe(f, v); fe_tobytes_words(w, f);
#pragma unroll
    for (int q = 0; q < 8; q++) w[q] = ok ? w[q] : (q == 0 ? c : 0u);
    o[0] = make_uint4(w[0], w[1], w[2], w[3]);
    o[1] = make_uint4(w[4], w[5], w[6], w[7]);
}
// Z of point i; returns 1 if it is non-zero mod p
__device__ __forceinline__ uint32_t load_z(fe64 &h, const uint64_t *__restrict__ in, size_t i)
{
    uint64_t l[5];
#pragma unroll
    for (int k = 0; k < 5; k++) l[k] = __ldg(in + 20 * i + 10 + k);
    fe t; fe_from_limbs51(t, l);
    fe64_from_fe_limbs(h, t);
    return 1u - (uint32_t)fe_iszero(t);
}
__device__ __forceinline__ void fe64_shfl_up(fe64 &o, const fe64 &f, int d)
{
#pragma unroll
    for (int k = 0; k < 5; k++) o.v[k] = __shfl_up_sync(0xffffffffu, f.v[k], d);
}
__device__ __forceinline__ void fe64_shfl_down(fe64 &o, const fe64 &f, int d)
{
#pragma unroll
    for (int k = 0; k < 5; k++) o.v[k] = __shfl_down_sync(0xffffffffu, f.v[k], d);
}
__device__ __forceinline__ void fe64_shfl_xor(fe64 &o, const fe64 &f, int m)
{
#pragma unroll
    for (int k = 0; k < 5; k++) o.v[k] = __shfl_xor_sync(0xffffffffu, f.v[k], m);
}
__device__ __forceinline__ void fe64_shfl_idx(fe64 &o, const fe64 &f, int src)
{
#pragma unroll
    for (int k = 0; k < 5; k++) o.v[k] = __shfl_sync(0xffffffffu, f.v[k], src);
}

// p = the product of x over the first `width` lanes (a power of two), in each of them
__device__ __forceinline__ void warp_product(fe64 &p, const fe64 &x, int width)
{
    fe64 t;
    p = x;
#pragma unroll 1
    for (int m = width >> 1; m > 0; m >>= 1) { fe64_shfl_xor(t, p, m); fe64_mul(p, p, t); }
}

// Products of x over the other lanes of the warp: below = the lanes under this one, above = the lanes over it (1 if
// none), all = the whole warp's, in every lane
__device__ __forceinline__ void warp_other_products(const fe64 &x, fe64 &below, fe64 &above, fe64 &all)
{
    const uint32_t lane = threadIdx.x & 31;
    fe64 lo = x, hi = x, t;
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) {
        fe64_shfl_up(t, lo, d);
        if (lane >= (uint32_t)d) fe64_mul(lo, lo, t);
        fe64_shfl_down(t, hi, d);
        if (lane + d < 32) fe64_mul(hi, hi, t);
    }
    fe64_shfl_idx(all, lo, 31);
    fe64_shfl_up(below, lo, 1); if (lane == 0) fe64_1(below);
    fe64_shfl_down(above, hi, 1); if (lane == 31) fe64_1(above);
}

// Montgomery's trick across the CTA (blockDim.x a multiple of 32, at most 1024): every thread holds the product acc of
// its own elements (never zero); inv = 1 / acc.  Two levels of warp_other_products, the lanes of each warp and then
// the warp products in warp 0, around one inversion of the CTA's product (INVERT: warp 0 inverts it) or none (its
// inverse is *tot_inv).  s_warp: one element per warp.
template <bool INVERT>
__device__ __forceinline__ void block_inverse(fe64 &inv, const fe64 &acc, fe64 *s_warp, const fe64 *tot_inv)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    fe64 below, above, all;
    warp_other_products(acc, below, above, all);
    if (lane == 0) s_warp[warp] = all;
    __syncthreads();
    if (warp == 0) {
        fe64 x, b, a, t;
        if (lane < nw) x = s_warp[lane]; else fe64_1(x);
        warp_other_products(x, b, a, all);
        if (INVERT) {   // limb-parallel on warp 0's lanes (warp4_f64.cuh): one lone thread's chain is latency-bound
            const w20_role r = w20_roles();
            const double inv = w20_invert(w20_limb(all, r.i), r);
#pragma unroll
            for (uint32_t k = 0; k < 5; k++) t.v[k] = w20_shfl(inv, k);
        } else {
            t = *tot_inv;
        }
        fe64_mul(t, t, b); fe64_mul(t, t, a);
        if (lane < nw) s_warp[lane] = t;
    }
    __syncthreads();
    fe64_mul(inv, s_warp[warp], below); fe64_mul(inv, inv, above);
}

// Pass 1: prod[g] = the product of the non-zero Z of group g
__global__ void __launch_bounds__(PREP_THREADS, 2)
k_prep_zprod(const uint64_t *__restrict__ in, fe64 *__restrict__ prod, size_t n)
{
    __shared__ fe64 s_warp[PREP_NW];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t g0 = (size_t)blockIdx.x * PREP_GROUP + tid;
    fe64 z[PREP_PER_THREAD], acc, t;
    uint32_t ok[PREP_PER_THREAD];
#pragma unroll
    for (int k = 0; k < PREP_PER_THREAD; k++) {           // every load is issued before the first multiplication
        const size_t i = g0 + (size_t)k * PREP_THREADS;
        if (i < n) ok[k] = load_z(z[k], in, i); else { ok[k] = 0; fe64_1(z[k]); }
    }
    acc = z[0];
    if (!ok[0]) fe64_1(acc);
#pragma unroll
    for (int k = 1; k < PREP_PER_THREAD; k++) { fe64_mul(t, acc, z[k]); fe64_cmov(acc, t, ok[k]); }
    warp_product(t, acc, 32);
    if (lane == 0) s_warp[warp] = t;
    __syncthreads();
    if (warp == 0) {
        if (lane < PREP_NW) acc = s_warp[lane]; else fe64_1(acc);
        warp_product(t, acc, PREP_NW);
        if (lane == 0) prod[blockIdx.x] = t;
    }
}

// Pass 2, one CTA: prod[g] <- 1 / prod[g] for all G groups.  Thread t takes a run of consecutive products
// (running products in pre[]), and block_inverse makes the one inversion.
__global__ void __launch_bounds__(PREP_THREADS)
k_prep_invert(fe64 *__restrict__ prod, fe64 *__restrict__ pre, uint32_t G)
{
    __shared__ fe64 s_warp[PREP_NW];
    const uint32_t per = (G + blockDim.x - 1) / blockDim.x, b = min(threadIdx.x * per, G), e = min(b + per, G);
    fe64 acc, inv, t;
    fe64_1(acc);
    for (uint32_t k = b; k < e; k++) { fe64_mul(acc, acc, prod[k]); pre[k] = acc; }
    block_inverse<true>(inv, acc, s_warp, nullptr);
    for (uint32_t k = e; k-- > b;) {                      // invariant: inv = 1 / pre[k]
        const fe64 x = prod[k];
        if (k > b) fe64_mul(t, inv, pre[k - 1]); else t = inv;
        prod[k] = t;
        fe64_mul(inv, inv, x);
    }
}

// Pass 3: every point of group g from the group's inverse ginv[g]
__global__ void __launch_bounds__(PREP_THREADS, 2)
k_prep_finish(const uint64_t *__restrict__ in, const fe64 *__restrict__ ginv, ge_niels_packed *__restrict__ out, size_t n)
{
    __shared__ fe64 s_warp[PREP_NW];
    __shared__ fe64 s_pre[PREP_PER_THREAD - 1][PREP_THREADS];   // running products but the last, kept out of the registers
    const uint32_t tid = threadIdx.x;
    const size_t g0 = (size_t)blockIdx.x * PREP_GROUP + tid;
    // running products pre[k] = Z_0 ... Z_k of this thread's points (zeros and points past n skipped)
    fe64 acc, inv;
    uint32_t nz = 0;                                       // bit k: Z_k != 0
    fe64_1(acc);
#pragma unroll 1
    for (int k = 0; k < PREP_PER_THREAD; k++) {
        const size_t i = g0 + (size_t)k * PREP_THREADS;
        if (k > 0) s_pre[k - 1][tid] = acc;
        if (i < n) {
            fe64 z, t;
            const uint32_t ok = load_z(z, in, i);
            fe64_mul(t, acc, z); fe64_cmov(acc, t, ok);
            nz |= ok << k;
        }
    }
    block_inverse<false>(inv, acc, s_warp, ginv + blockIdx.x);   // 1 / pre[PREP_PER_THREAD - 1]
#pragma unroll 1
    for (int k = PREP_PER_THREAD - 1; k >= 0; k--) {       // invariant: inv = 1 / pre[k]
        const size_t i = g0 + (size_t)k * PREP_THREADS;
        if (i >= n) continue;
        const uint32_t ok = (nz >> k) & 1u;
        const uint64_t *src = in + 20 * i;
        fe64 X, Y, zi, u, v;
        load_coord_f64(u, src + 10);                       // Z_k again (the forward loop above read it)
        if (k > 0) fe64_mul(zi, inv, s_pre[k - 1][tid]); else zi = inv;   // 1 / Z_k
        fe64_mul(v, inv, u); fe64_cmov(inv, v, ok);
        // each coordinate goes to its canonical bytes, and out, as soon as it is made (fewer live registers); Z = 0
        // gives the identity (1, 1, 0)
        uint4 *o = reinterpret_cast<uint4 *>(out + i);
        load_coord_f64(X, src); load_coord_f64(Y, src + 5);
        fe64_add(u, Y, X); fe64_mul(v, u, zi);                         // 2 x 1
        store_coord(o, v, ok, 1u);
        fe64_sub(u, Y, X); fe64_mul(v, u, zi);
        store_coord(o + 2, v, ok, 1u);
        load_coord_f64(u, src + 15);
        fe64_mul(v, u, zi); fe64_const_2d(u); fe64_mul(v, v, u);
        store_coord(o + 4, v, ok, 0u);
    }
}

// Extended points -> projective Niels (Y+X, Y-X, Z, 2dT), no inversion: for the latency-bound vartime Straus path,
// which builds its own tables from the point
__global__ void k_prep_extended_pniels(const uint64_t *__restrict__ in, ge_pniels_packed *__restrict__ out, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(in + 20 * i);
    uint64_t l[20];
#pragma unroll
    for (int k = 0; k < 10; k++) { ulonglong2 v = src[k]; l[2 * k] = v.x; l[2 * k + 1] = v.y; }
    ge_p3 p;
    fe_from_limbs51(p.X, l); fe_from_limbs51(p.Y, l + 5); fe_from_limbs51(p.Z, l + 10); fe_from_limbs51(p.T, l + 15);
    ge_pniels pn; ge_p3_to_pniels(pn, p);
    ge_pniels_packed pk; ge_pniels_pack(pk, pn);
    uint4 *o = reinterpret_cast<uint4 *>(out + i);
#pragma unroll
    for (int k = 0; k < 8; k++) o[k] = make_uint4(pk.w[4 * k], pk.w[4 * k + 1], pk.w[4 * k + 2], pk.w[4 * k + 3]);
}

int msm_prepared_kind(int point_fmt, int kind)
{
    return point_fmt == DALEK_POINTS_EXTENDED ? kind : PK_NIELS;
}

int msm_prepare_points_on(dalek_b200_ctx *ctx, cudaStream_t st, const void *d_in, int point_fmt, size_t n, void *d_out, int *d_bad,
                          int kind)
{
    if (n == 0) return 0;
    if (point_fmt == DALEK_POINTS_COMPRESSED) {
        if (ctx->opt_decompress_f64) k_prep_compressed<1><<<cdiv(n, 128), 128, 0, st>>>((const uint4 *)d_in, (ge_niels_packed *)d_out, n, d_bad);
        else k_prep_compressed<0><<<cdiv(n, 128), 128, 0, st>>>((const uint4 *)d_in, (ge_niels_packed *)d_out, n, d_bad);
    } else if (point_fmt == DALEK_POINTS_RISTRETTO) {
        if (ctx->opt_decompress_f64) k_prep_ristretto<1><<<cdiv(n, 128), 128, 0, st>>>((const uint32_t *)d_in, (ge_niels_packed *)d_out, n, d_bad);
        else k_prep_ristretto<0><<<cdiv(n, 128), 128, 0, st>>>((const uint32_t *)d_in, (ge_niels_packed *)d_out, n, d_bad);
    } else if (kind == PK_PNIELS) {
        k_prep_extended_pniels<<<cdiv(n, 128), 128, 0, st>>>((const uint64_t *)d_in, (ge_pniels_packed *)d_out, n);
    } else {
        // one workspace per context: the calls that prepare points (one per chunk of a host-buffer call) follow each
        // other on one stream
        const unsigned G = cdiv(n, PREP_GROUP);
        int rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_PREP_PROD], 2 * (size_t)G * sizeof(fe64)))) return rc;
        fe64 *prod = (fe64 *)ctx->ws[WS_PREP_PROD].p;
        k_prep_zprod<<<G, PREP_THREADS, 0, st>>>((const uint64_t *)d_in, prod, n);
        k_prep_invert<<<1, PREP_THREADS, 0, st>>>(prod, prod + G, G);
        k_prep_finish<<<G, PREP_THREADS, 0, st>>>((const uint64_t *)d_in, prod, (ge_niels_packed *)d_out, n);
        ctx->launches += 2;
    }
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

int msm_prepare_points(dalek_b200_ctx *ctx, const void *d_in, int point_fmt, size_t n, void *d_out, int *d_bad, int kind)
{
    return msm_prepare_points_on(ctx, ctx->stream, d_in, point_fmt, n, d_out, d_bad, kind);
}

// ------------------------------------------------------------------------------------------
// window selection: minimise windows * (n + ~2.5 * buckets) (bucket adds + reduction adds)
int msm_window_count_for_bits(int c) { return 256 / c + 1; }

int msm_choose_window_bits(const dalek_b200_ctx *ctx, size_t n)
{
    if (ctx->opt_window_bits >= 4 && ctx->opt_window_bits <= 20) return (int)ctx->opt_window_bits;
    int best = 4; double best_cost = 1e300;
    for (int c = 4; c <= 20; c++) {
        double W = (double)((253 + c - 1) / c);
        double cost = W * ((double)n + 4.0 * (double)(1u << (c - 1)));
        if (cost < best_cost) { best_cost = cost; best = c; }
    }
    return best;
}

// The same cost model when `n_short` scalars have only `short_bits` bits: they contribute ceil((bits+1)/c)
// bucket additions each (one spare bit for the signed-digit carry).
int msm_choose_window_bits_mixed(const dalek_b200_ctx *ctx, size_t n_short, int short_bits, size_t n_long)
{
    if (ctx->opt_window_bits >= 4 && ctx->opt_window_bits <= 20) return (int)ctx->opt_window_bits;
    int best = 4; double best_cost = 1e300;
    for (int c = 4; c <= 20; c++) {
        double W = (double)((253 + c - 1) / c), Ws = (double)((short_bits + 1 + c - 1) / c);
        double cost = Ws * (double)n_short + W * ((double)n_long + 4.0 * (double)(1u << (c - 1)));
        if (cost < best_cost) { best_cost = cost; best = c; }
    }
    return best;
}

// ------------------------------------------------------------------------------------------
// Counting sort of the digits by (window, bucket), two levels.  A coarse bin is 2^F consecutive buckets of one
// bucket window (F = fine bits, msm_sort_fine_bits).
//   k_sort_count      one CTA per tile of SORT_COUNT_TILE scalars: shared histogram over (window, coarse bin), one
//                     global atomic per non-empty bin
//   k_sort_bins_scan  one CTA per bucket window: exclusive scan of its coarse counts -> bin cursors
//   k_sort_partition  one CTA per tile of SORT_TILE scalars, window by window: the tile's records are staged in
//                     shared memory by coarse bin, one atomic per (tile, bin) reserves a run of the bin, and the
//                     runs are written contiguously.  Record = (stored index | sign << 31, fine digit), 8 B.
//   k_sort_fine       one CTA per coarse bin (per slice of SORT_FINE_CAP records of a bigger one): counting sort on
//                     the low F bits in shared memory; writes the bin's counts, offsets and sorted entries
// Every scattered store lands in shared memory; global memory sees runs and whole bins.  The order of the entries
// inside a bucket depends on the order of the atomics: the bucket sums are the same group elements either way.
// flat != 0 (a table stride): the digits of every window count into the buckets of window 0 (precomputed 2^(cw) P
// tables) and the stored index is w * flat + i.
#define SORT_THREADS 512
#define SORT_COUNT_TILE 4096u     // scalars per CTA of k_sort_count
#define SORT_TILE 2048u           // scalars per CTA of k_sort_partition (SORT_TILE / SORT_THREADS per thread)
#define SORT_HIST_MAX 8192u       // (window, coarse bin) counters of one k_sort_count CTA
#define SORT_NC_MAX 4096u         // coarse bins per window
#define SORT_FINE_MAX 12          // fine bits
#define SORT_BIN_MEAN 4096u       // coarse bins are added while their mean size on uniform digits is above this
#define SORT_FINE_CAP 8192u       // records of a coarse bin (or of a slice of a bigger one) k_sort_fine holds in shared memory
// Dynamic shared memory of the two sort kernels at the largest nc and F msm_sort_fine_bits can pick (49284 B and
// 114820 B).  The limit a launch is checked against belongs to the kernel on the device, not to a context: a per-call
// value set by one context would lower the limit under a concurrent call of another context with a larger nc or F.
// So every context sets these call-independent bounds once, and each launch passes its own, smaller size.
#define SORT_PART_SMEM_MAX (SORT_TILE * 8 + (2 * SORT_NC_MAX + 33) * 4)
#define SORT_FINE_SMEM_MAX (SORT_FINE_CAP * 12 + ((1u << SORT_FINE_MAX) + 33) * 4)

// Digit of the lowest remaining window of s (tests/msm_digit_cases.py): s is shifted right by c, carry in and out.
__device__ __forceinline__ int32_t next_digit(uint32_t s[8], uint32_t &carry, int c)
{
    const uint32_t v = (s[0] & ((1u << c) - 1)) + carry;
#pragma unroll
    for (int k = 0; k < 7; k++) s[k] = __funnelshift_r(s[k], s[k + 1], c);
    s[7] >>= c;
    if (v > (1u << (c - 1))) { carry = 1; return (int32_t)v - (int32_t)(1u << c); }
    carry = 0;
    return (int32_t)v;
}

__device__ __forceinline__ void load_scalar(uint32_t s[8], const uint4 *__restrict__ scalars, size_t i)
{
    const uint4 a = scalars[2 * i], b = scalars[2 * i + 1];
    s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
}

// In-place exclusive scan of v[0, len) in shared memory by the whole CTA; returns the total.  scr: 33 words.
__device__ uint32_t block_excl_scan(uint32_t *v, uint32_t len, uint32_t *scr)
{
    const uint32_t t = threadIdx.x, lane = t & 31, wid = t >> 5, nw = blockDim.x >> 5;
    const uint32_t per = (len + blockDim.x - 1) / blockDim.x, b = min(t * per, len), e = min(b + per, len);
    __syncthreads();
    uint32_t sum = 0;
    for (uint32_t k = b; k < e; k++) sum += v[k];
    uint32_t incl = sum;
    for (int d = 1; d < 32; d <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += x; }
    if (lane == 31) scr[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const uint32_t x = lane < nw ? scr[lane] : 0;
        uint32_t y = x;
        for (int d = 1; d < 32; d <<= 1) { uint32_t z = __shfl_up_sync(0xffffffffu, y, d); if (lane >= (uint32_t)d) y += z; }
        if (lane < nw) scr[lane] = y - x;
        if (lane == 31) scr[32] = y;
    }
    __syncthreads();
    uint32_t run = scr[wid] + incl - sum;
    for (uint32_t k = b; k < e; k++) { const uint32_t x = v[k]; v[k] = run; run += x; }
    const uint32_t total = scr[32];
    __syncthreads();
    return total;
}

// Position inside ctr[key] for every live lane of the warp, one atomic per distinct key: the big bins that
// k_sort_partition counts and k_sort_fine slices come from skewed digits, where most lanes share a key.  Every lane
// of the warp must call it.
__device__ __forceinline__ uint32_t warp_claim(uint32_t *ctr, uint32_t key, bool live)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t peers = __match_any_sync(0xffffffffu, live ? key : 0xffffffffu);
    const uint32_t leader = __ffs(peers) - 1;
    uint32_t base = 0;
    if (live && lane == leader) base = atomicAdd(&ctr[key], (uint32_t)__popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    return base + __popc(peers & ((1u << lane) - 1));
}

__global__ void __launch_bounds__(SORT_THREADS)
k_sort_count(const uint4 *__restrict__ scalars, size_t n, int c, int nact, int F, uint32_t nc, int flat,
             uint32_t *__restrict__ ccount)
{
    __shared__ uint32_t h[SORT_HIST_MAX];
    const uint32_t nh = (flat ? 1u : (uint32_t)nact) * nc;
    for (uint32_t k = threadIdx.x; k < nh; k += SORT_THREADS) h[k] = 0;
    __syncthreads();
    for (uint32_t j = 0; j < SORT_COUNT_TILE / SORT_THREADS; j++) {
        const size_t i = (size_t)blockIdx.x * SORT_COUNT_TILE + j * SORT_THREADS + threadIdx.x;
        if (i >= n) break;
        uint32_t s[8], carry = 0;
        load_scalar(s, scalars, i);
        for (int w = 0; w < nact; w++) {
            const int32_t d = next_digit(s, carry, c);
            if (d) atomicAdd(&h[(flat ? 0u : (uint32_t)w * nc) + (((uint32_t)(d < 0 ? -d : d) - 1) >> F)], 1u);
        }
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < nh; k += SORT_THREADS)
        if (h[k]) atomicAdd(&ccount[k], h[k]);
}

// A coarse bin of more than SORT_FINE_CAP records (skewed scalars; the short scalars of verify_batch put half of
// their digits of one window into one bucket) is "big": k_sort_partition counts its buckets with global atomics and
// k_sort_fine sorts it in slices of SORT_FINE_CAP records, one CTA per slice.  Slice 0 of every bin runs in CTA
// [0, nbins); the further slices ("extra") in CTAs nbins + the bin's place in the extra-slice prefix.
__device__ __forceinline__ uint32_t extra_slices(uint32_t cnt) { return cnt > SORT_FINE_CAP ? (cnt - 1) / SORT_FINE_CAP : 0; }

// One CTA per bucket window: cursor = exclusive scan of the coarse counts (bin bases inside the window's segment),
// xpre = exclusive scan of the bins' extra slices, xtot[w] = the window's extra slices.  The bucket counts and the
// fill counters of big bins are zeroed here, ahead of the atomics of k_sort_partition and k_sort_fine.
__global__ void __launch_bounds__(SORT_THREADS)
k_sort_bins_scan(const uint32_t *__restrict__ ccount, uint32_t nc, int F, uint32_t nbuckets, uint32_t *__restrict__ ccursor,
                 uint32_t *__restrict__ xpre, uint32_t *__restrict__ xtot, uint32_t *__restrict__ counts,
                 uint32_t *__restrict__ fill)
{
    __shared__ uint32_t v[SORT_NC_MAX], scr[33];
    const size_t o = (size_t)blockIdx.x * nc;
    for (uint32_t k = threadIdx.x; k < nc; k += SORT_THREADS) v[k] = ccount[o + k];
    block_excl_scan(v, nc, scr);
    for (uint32_t k = threadIdx.x; k < nc; k += SORT_THREADS) { ccursor[o + k] = v[k]; v[k] = extra_slices(ccount[o + k]); }
    const uint32_t total = block_excl_scan(v, nc, scr);
    for (uint32_t k = threadIdx.x; k < nc; k += SORT_THREADS) xpre[o + k] = v[k];
    if (threadIdx.x == 0) xtot[blockIdx.x] = total;
    for (uint32_t k = 0; k < nc; k++) {
        if ((k + 1 < nc ? v[k + 1] : total) == v[k]) continue;   // no extra slice: not big
        const size_t b0 = (size_t)blockIdx.x * nbuckets + ((size_t)k << F);
        for (uint32_t f = threadIdx.x; f < (1u << F); f += SORT_THREADS) { counts[b0 + f] = 0; fill[b0 + f] = 0; }
    }
}

// dynamic shared memory: stage[SORT_TILE] (uint2) | cnt[nc] | gbase[nc] | scr[33]
__global__ void __launch_bounds__(SORT_THREADS, 2)
k_sort_partition(const uint4 *__restrict__ scalars, size_t n, int c, int nact, int F, uint32_t nc, uint32_t nbuckets, size_t flat,
                 const uint32_t *__restrict__ ccount, uint32_t *__restrict__ ccursor, uint2 *__restrict__ records,
                 uint32_t *__restrict__ counts)
{
    constexpr int SPT = SORT_TILE / SORT_THREADS;
    extern __shared__ uint32_t sm[];
    uint2 *stage = reinterpret_cast<uint2 *>(sm);
    uint32_t *cnt = sm + 2 * SORT_TILE, *gbase = cnt + nc, *scr = gbase + nc;
    const uint32_t fmask = (1u << F) - 1;
    uint32_t s[SPT][8], carry[SPT];
    size_t idx[SPT];
#pragma unroll
    for (int j = 0; j < SPT; j++) {
        idx[j] = (size_t)blockIdx.x * SORT_TILE + j * SORT_THREADS + threadIdx.x;
        carry[j] = 0;
        if (idx[j] < n) load_scalar(s[j], scalars, idx[j]);
        else for (int k = 0; k < 8; k++) s[j][k] = 0;          // zero digits: no record
    }
    for (int w = 0; w < nact; w++) {
        const uint32_t wb = flat ? 0u : (uint32_t)w;           // bucket window
        for (uint32_t k = threadIdx.x; k < nc; k += SORT_THREADS) cnt[k] = 0;
        __syncthreads();
        uint32_t bkt[SPT], rank[SPT], neg[SPT];
#pragma unroll
        for (int j = 0; j < SPT; j++) {
            const int32_t d = next_digit(s[j], carry[j], c);
            neg[j] = d < 0;
            bkt[j] = d ? (uint32_t)(d < 0 ? -d : d) - 1 : 0xffffffffu;
            if (d) rank[j] = atomicAdd(&cnt[bkt[j] >> F], 1u);
        }
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < nc; k += SORT_THREADS) {
            const uint32_t v = cnt[k];
            gbase[k] = v ? atomicAdd(&ccursor[(size_t)wb * nc + k], v) : 0;
        }
        const uint32_t total = block_excl_scan(cnt, nc, scr);  // cnt -> first staged slot of each bin
#pragma unroll
        for (int j = 0; j < SPT; j++) {
            if (bkt[j] == 0xffffffffu) continue;
            const uint32_t cb = bkt[j] >> F;
            const uint32_t val = (flat ? (uint32_t)((size_t)w * flat + idx[j]) : (uint32_t)idx[j]) | (neg[j] << 31);
            stage[cnt[cb] + rank[j]] = make_uint2(val, (bkt[j] & fmask) | (cb << 16));
        }
        __syncthreads();
        uint2 *dst = records + (flat ? (size_t)0 : (size_t)w * n);
        for (uint32_t k0 = 0; k0 < total; k0 += SORT_THREADS) {      // uniform trip count: warp_claim below
            const uint32_t k = k0 + threadIdx.x;
            const uint2 r = k < total ? stage[k] : make_uint2(0, 0);
            const uint32_t cb = r.y >> 16, f = r.y & 0xffffu;
            if (k < total) dst[gbase[cb] + (k - cnt[cb])] = make_uint2(r.x, f);
            const bool big = k < total && ccount[(size_t)wb * nc + cb] > SORT_FINE_CAP;
            if (__any_sync(0xffffffffu, big)) warp_claim(counts + (size_t)wb * nbuckets, (cb << F) | f, big);
        }
        __syncthreads();
    }
}

// Slice 0 of every coarse bin in CTAs [0, nbins), the top windows first (the skewed bins of reduced scalars and of short
// scalars are there); the extra slices of big bins after them.  The partition left ccursor at the end of the bin.
// A bin of at most SORT_FINE_CAP records is counted and sorted in shared memory and written out coalesced.  A slice
// of a big bin takes the bin's offsets from its complete counts, claims a run of each of its fine buckets with one
// atomic on the bucket's fill counter, and places its records in shared memory.
// dynamic shared memory: recs[SORT_FINE_CAP] (uint2) | out[SORT_FINE_CAP] | h[2^F] | scr[33]
__global__ void __launch_bounds__(SORT_THREADS, 2)
k_sort_fine(const uint2 *__restrict__ records, const uint32_t *__restrict__ ccount, const uint32_t *__restrict__ ccursor,
            const uint32_t *__restrict__ xpre, const uint32_t *__restrict__ xtot, size_t n, int F, uint32_t nc,
            uint32_t nbuckets, uint32_t nwin, int flat, uint32_t *__restrict__ counts, uint32_t *__restrict__ offsets,
            uint32_t *__restrict__ sorted, uint32_t *__restrict__ fill)
{
    extern __shared__ uint32_t sm[];
    __shared__ uint32_t s_bin, s_slice;
    uint2 *recs = reinterpret_cast<uint2 *>(sm);
    uint32_t *out = sm + 2 * SORT_FINE_CAP, *h = out + SORT_FINE_CAP, *scr = h + (1u << F);
    const uint32_t nf = 1u << F, nbins = nwin * nc;
    uint32_t bin, slice = 0;
    if (blockIdx.x < nbins) {
        bin = nbins - 1 - blockIdx.x;
    } else {
        if (threadIdx.x == 0) {
            uint32_t t = blockIdx.x - nbins, w = 0;
            while (w < nwin && t >= xtot[w]) t -= xtot[w++];
            s_bin = nbins;                                  // past the last extra slice
            if (w < nwin) {
                const uint32_t *x = xpre + (size_t)w * nc;
                uint32_t lo = 0, hi = nc - 1;               // the big bin: the last one with x[k] <= t
                while (lo < hi) { const uint32_t mid = (lo + hi + 1) / 2; if (x[mid] <= t) lo = mid; else hi = mid - 1; }
                s_bin = w * nc + lo;
                s_slice = t - x[lo] + 1;
            }
        }
        __syncthreads();
        bin = s_bin; slice = s_slice;
        if (bin >= nbins) return;
    }
    const uint32_t wb = bin / nc, cb = bin % nc;
    const uint32_t cnt = ccount[bin], base = ccursor[bin] - cnt;
    const size_t seg = flat ? (size_t)0 : (size_t)wb * n;
    const size_t b0 = (size_t)wb * nbuckets + ((size_t)cb << F);
    const uint2 *src = records + seg + base;
    uint32_t *dst = sorted + seg + base;
    constexpr uint32_t U = 4;                               // records in flight per thread
    if (cnt <= SORT_FINE_CAP) {
        for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) h[f] = 0;
        __syncthreads();
        for (uint32_t k0 = 0; k0 < cnt; k0 += U * SORT_THREADS) {
            uint2 r[U];
#pragma unroll
            for (uint32_t u = 0; u < U; u++) {
                const uint32_t k = k0 + u * SORT_THREADS + threadIdx.x;
                r[u] = k < cnt ? src[k] : make_uint2(0, 0);
            }
#pragma unroll
            for (uint32_t u = 0; u < U; u++) {
                const uint32_t k = k0 + u * SORT_THREADS + threadIdx.x;
                if (k < cnt) { recs[k] = r[u]; atomicAdd(&h[r[u].y], 1u); }
            }
        }
        __syncthreads();
        for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) counts[b0 + f] = h[f];
        block_excl_scan(h, nf, scr);
        for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) offsets[b0 + f] = base + h[f];
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < cnt; k += SORT_THREADS) { const uint2 r = recs[k]; out[atomicAdd(&h[r.y], 1u)] = r.x; }
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < cnt; k += SORT_THREADS) dst[k] = out[k];
        return;
    }
    // a slice of a big bin; out[0, nf) = the slice's counts, then the positions of its runs in the bin
    for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) { h[f] = counts[b0 + f]; out[f] = 0; }
    block_excl_scan(h, nf, scr);
    if (slice == 0)
        for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) offsets[b0 + f] = base + h[f];
    const uint32_t lo = slice * SORT_FINE_CAP, m = min(SORT_FINE_CAP, cnt - lo);
    for (uint32_t k0 = 0; k0 < m; k0 += U * SORT_THREADS) {
        uint2 r[U];
#pragma unroll
        for (uint32_t u = 0; u < U; u++) {
            const uint32_t k = k0 + u * SORT_THREADS + threadIdx.x;
            r[u] = k < m ? src[lo + k] : make_uint2(0, 0);
        }
#pragma unroll
        for (uint32_t u = 0; u < U; u++) {
            const uint32_t k = k0 + u * SORT_THREADS + threadIdx.x;
            if (k < m) recs[k] = r[u];
            warp_claim(out, r[u].y, k < m);
        }
    }
    __syncthreads();
    for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS)
        if (out[f]) out[f] = h[f] + atomicAdd(&fill[b0 + f], out[f]);
    __syncthreads();
    for (uint32_t k0 = 0; k0 < m; k0 += SORT_THREADS) {
        const uint32_t k = k0 + threadIdx.x;
        const uint2 r = k < m ? recs[k] : make_uint2(0, 0);
        const uint32_t pos = warp_claim(out, r.y, k < m);
        if (k < m) dst[pos] = r.x;
    }
}

// per-window exclusive scan of the task counts -> task list offsets (relative to the window's list), multi-block:
// k_scan_partial (sum of each 4096-entry part), k_scan_bases (exclusive scan of the part sums of a
// window, one CTA per window), k_scan_apply (local scan + part base).
#define SCAN_PART 4096u
__global__ void __launch_bounds__(1024) k_scan_partial(const uint32_t *__restrict__ in, uint32_t nbuckets, uint32_t parts,
                                                       uint32_t *__restrict__ part_sums)
{
    __shared__ uint32_t sh[32];
    uint32_t w = blockIdx.x / parts, part = blockIdx.x % parts;
    const uint32_t *src = in + (size_t)w * nbuckets;
    uint32_t base = part * SCAN_PART + threadIdx.x * 4, sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) if (base + k < nbuckets) sum += src[base + k];
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, d);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t v = sh[threadIdx.x];
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
        if (threadIdx.x == 0) part_sums[blockIdx.x] = v;
    }
}
__global__ void k_scan_bases(uint32_t *__restrict__ part_sums, uint32_t parts)
{
    // one CTA (one thread is enough: parts <= 128) per window: in-place exclusive scan
    if (threadIdx.x) return;
    uint32_t *p = part_sums + (size_t)blockIdx.x * parts, run = 0;
    for (uint32_t k = 0; k < parts; k++) { uint32_t v = p[k]; p[k] = run; run += v; }
}
__global__ void __launch_bounds__(1024) k_scan_apply(const uint32_t *__restrict__ in, const uint32_t *__restrict__ part_base,
                                                     uint32_t nbuckets, uint32_t parts, uint32_t *__restrict__ out)
{
    __shared__ uint32_t sh[32];
    uint32_t w = blockIdx.x / parts, part = blockIdx.x % parts;
    const uint32_t *src = in + (size_t)w * nbuckets;
    uint32_t *dst = out + (size_t)w * nbuckets;
    uint32_t base = part * SCAN_PART + threadIdx.x * 4;
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) { v[k] = base + k < nbuckets ? src[base + k] : 0; sum += v[k]; }
    uint32_t incl = sum;                                   // inclusive scan of thread sums inside the warp
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if ((threadIdx.x & 31) >= d) incl += t; }
    if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t x = sh[threadIdx.x], inc2 = x;
        for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc2, d); if (threadIdx.x >= d) inc2 += t; }
        sh[threadIdx.x] = inc2 - x;                        // exclusive warp bases
    }
    __syncthreads();
    uint32_t run = part_base[blockIdx.x] + sh[threadIdx.x >> 5] + incl - sum;
#pragma unroll
    for (int k = 0; k < 4; k++) { if (base + k < nbuckets) dst[base + k] = run; run += v[k]; }
}

// ------------------------------------------------------------------------------------------
// Bucket accumulation as a list of tasks.  A task is at most task_len consecutive entries of one
// bucket; a bucket with more entries (skewed inputs: the 128-bit z_i of verify_batch put n/256
// points into each of 256 buckets of one window; adversarial inputs can put everything into one)
// is cut into several tasks whose partial sums are added afterwards by k_heavy_fixup.
// task_len (msm_task_len) is twice the mean bucket size when the buckets alone give enough parallelism,
// so that only genuinely skewed buckets are cut; with few buckets it is what yields >= 2^18 tasks.
#define TASK_LEN_MIN 64u
static uint32_t msm_task_len(size_t n, int nwin, uint32_t nb)
{
    const size_t total_buckets = (size_t)nwin * nb;
    const size_t want = total_buckets >= ((size_t)1 << 18) ? 2 * (n / nb) : (n * (size_t)nwin) >> 18;
    uint32_t len = TASK_LEN_MIN;
    while (len < want && len < (1u << 22)) len <<= 1;
    return len;
}
#ifndef ACC_MIN_BLOCKS
#define ACC_MIN_BLOCKS 4
#endif

// also appends every bucket that needs more than one task to the heavy list (heavy[0] = count)
__global__ void k_task_count(const uint32_t *__restrict__ counts, uint32_t total_buckets, uint32_t task_len,
                             uint32_t *__restrict__ ntasks, uint32_t *__restrict__ heavy)
{
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total_buckets) return;
    uint32_t c = counts[t];
    uint32_t k = c <= task_len ? 1u : (c + task_len - 1) / task_len;
    ntasks[t] = k;
    if (k > 1) heavy[1 + atomicAdd(&heavy[0], 1u)] = t;
}

// per-window bases of the task lists (exclusive prefix over windows) and the grand total
__global__ void k_task_bases(const uint32_t *__restrict__ ntasks, const uint32_t *__restrict__ task_off, uint32_t nbuckets,
                             int nwin, uint32_t *__restrict__ win_base /* nwin + 1 */)
{
    if (blockIdx.x || threadIdx.x) return;
    uint32_t run = 0;
    for (int w = 0; w < nwin; w++) {
        win_base[w] = run;
        size_t last = (size_t)w * nbuckets + nbuckets - 1;
        run += task_off[last] + ntasks[last];
    }
    win_base[nwin] = run;
}

// task p = (bucket t, piece j) stored as two u32
__global__ void k_task_fill(const uint32_t *__restrict__ ntasks, const uint32_t *__restrict__ task_off,
                            const uint32_t *__restrict__ win_base, uint32_t nbuckets, uint32_t total_buckets,
                            uint2 *__restrict__ tasks)
{
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total_buckets) return;
    uint32_t w = t / nbuckets;
    uint32_t base = win_base[w] + task_off[t], k = ntasks[t];
    for (uint32_t j = 0; j < k; j++) tasks[base + j] = make_uint2(t, j);
}

// Tasks are processed in order of decreasing length (counting sort on the quantised length, TASK_BINS bins):
// the lanes of a warp then run the same trip count, and the grid drains longest-first, so the kernel does not
// end on a few long tasks.  order[q] = task index; hist | cursor | start are TASK_BINS words each.
#define TASK_BINS 256u
__device__ __forceinline__ uint32_t task_key(uint32_t len, uint32_t task_len)
{
    return (uint32_t)(((uint64_t)len * (TASK_BINS - 1) + task_len - 1) / task_len);     // 0 only for an empty task
}
__device__ __forceinline__ uint32_t task_length(const uint2 tk, const uint32_t *__restrict__ counts, uint32_t task_len)
{
    return min(task_len, counts[tk.x] - tk.y * task_len);
}

__global__ void __launch_bounds__(256)
k_task_hist(const uint2 *__restrict__ tasks, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ total_ptr,
            uint32_t task_len, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t sh[TASK_BINS];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < *total_ptr) atomicAdd(&sh[task_key(task_length(tasks[p], counts, task_len), task_len)], 1u);
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

// start[k] = number of tasks with a larger key
__global__ void __launch_bounds__(256) k_task_scan(const uint32_t *__restrict__ hist, uint32_t *__restrict__ start)
{
    __shared__ uint32_t sh[TASK_BINS];
    const uint32_t k = TASK_BINS - 1 - threadIdx.x;              // thread 0 holds the largest key
    sh[threadIdx.x] = hist[k];
    __syncthreads();
    for (uint32_t d = 1; d < TASK_BINS; d <<= 1) {
        uint32_t v = threadIdx.x >= d ? sh[threadIdx.x - d] : 0;
        __syncthreads();
        sh[threadIdx.x] += v;
        __syncthreads();
    }
    start[k] = sh[threadIdx.x] - hist[k];
}

__global__ void __launch_bounds__(256)
k_task_scatter(const uint2 *__restrict__ tasks, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ total_ptr,
               uint32_t task_len, const uint32_t *__restrict__ start, uint32_t *__restrict__ cursor, uint32_t *__restrict__ order)
{
    __shared__ uint32_t cnt[TASK_BINS], base[TASK_BINS];
    cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < *total_ptr;
    uint32_t key = 0, rank = 0;
    if (live) { key = task_key(task_length(tasks[p], counts, task_len), task_len); rank = atomicAdd(&cnt[key], 1u); }
    __syncthreads();
    if (cnt[threadIdx.x]) base[threadIdx.x] = start[threadIdx.x] + atomicAdd(&cursor[threadIdx.x], cnt[threadIdx.x]);
    __syncthreads();
    if (live) order[base[key] + rank] = p;
}

__device__ __forceinline__ void load_p3(ge_p3 &p, const ge_p3_raw *src)
{
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    ge_p3_raw r;
#pragma unroll
    for (int q = 0; q < 10; q++) { uint4 v = s[q]; r.w[4 * q] = v.x; r.w[4 * q + 1] = v.y; r.w[4 * q + 2] = v.z; r.w[4 * q + 3] = v.w; }
    ge_p3_load_raw(p, r);
}

// TMA = 1: the gather of the next point is ONE bulk copy of the TMA unit (cp.async.bulk.shared.global, completion
// on a per-thread mbarrier) instead of 6 16-byte cp.async (LDGSTS); tools/ab_tma.py is the A/B measurement.
template <int F64, int TMA>
__global__ void __launch_bounds__(128, ACC_MIN_BLOCKS)
k_bucket_accumulate(const ge_niels_packed *__restrict__ points, const uint32_t *__restrict__ sorted,
                    const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offsets,
                    const uint32_t *__restrict__ ntasks, const uint2 *__restrict__ tasks, const uint32_t *__restrict__ order,
                    const uint32_t *__restrict__ win_base, int w0, int w1, size_t n, uint32_t nbuckets, uint32_t task_len,
                    ge_p3_raw *__restrict__ buckets, ge_p3_raw *__restrict__ task_sums, int first)
{
    constexpr int NQ = sizeof(ge_niels_packed) / 16;          // 16-byte pieces per point
    constexpr int TSTRIDE = NQ * 16 + 16;                     // bulk copies land contiguously: pad the per-thread slot so
                                                              // that the 16-byte reads of 8 consecutive threads hit 8 different bank groups
    __shared__ uint4 s_pts[(F64 && !TMA) ? 2 : 1][(F64 && !TMA) ? NQ : 1][(F64 && !TMA) ? 128 : 1];   // cp.async slots, [buffer][piece][thread]: conflict-free
    __shared__ __align__(16) unsigned char s_bulk[(F64 && TMA) ? 2 : 1][(F64 && TMA) ? 128 : 1][(F64 && TMA) ? TSTRIDE : 16];
    __shared__ __align__(8) unsigned long long s_bar[(F64 && TMA) ? 2 : 1][(F64 && TMA) ? 128 : 1];
    const uint32_t total_tasks = win_base[w1];            // this launch covers the tasks of windows [w0, w1)
    const uint32_t slot = blockIdx.x * 128u + threadIdx.x;
    if (slot >= total_tasks) return;
    const uint32_t p = order[slot];                        // tasks in order of decreasing length
    const uint2 tk = tasks[p];
    const uint32_t t = tk.x, w = t / nbuckets;
    const uint32_t cnt = counts[t], start = tk.y * task_len;
    const uint32_t len = min(task_len, cnt - start);
    // `first` = first chunk of points: buckets start at the identity.  Later chunks (host inputs are
    // streamed in chunks so that the copies overlap the arithmetic) add onto the stored bucket sums;
    // the stored sum is folded in by piece 0 of the bucket (or by k_heavy_fixup for split buckets).
    const bool split = ntasks[t] != 1;
    if (!first && len == 0) return;                        // nothing new for this bucket
    const bool fold_old = !first && !split;
    const uint32_t *idx = sorted + (size_t)w * n + offsets[t] + start;
    ge_p3 acc;
    if (F64) {
        // FP64-pipe field (fe64.cuh): 1.65x the multiplication rate of the IMAD.WIDE form
        // The gather of the NEXT point (into this thread's shared-memory slot, two slots per thread) is in flight
        // while the current addition runs, so the HBM/L2 latency of the random gathers is off the dependent path.
        ge64_p3 acc64;
        if (fold_old) {
            ge_p3 old; load_p3(old, buckets + t);
            fe64_from_fe(acc64.X, old.X); fe64_from_fe(acc64.Y, old.Y); fe64_from_fe(acc64.Z, old.Z); fe64_from_fe(acc64.T, old.T);
        } else {
            ge64_identity(acc64);
        }
        uint32_t e_next = len ? idx[0] : 0;
        if (TMA) {
            const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&s_bar[0][threadIdx.x]);
            const uint32_t bar1 = (uint32_t)__cvta_generic_to_shared(&s_bar[1][threadIdx.x]);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0) : "memory");
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar1) : "memory");
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        auto prefetch = [&](uint32_t e, int buf) {
            const uint32_t pi = e & 0x7fffffffu;
            const char *src = reinterpret_cast<const char *>(points) + (size_t)pi * (NQ * 16);
            if (TMA) {
                const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&s_bar[buf][threadIdx.x]);
                const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&s_bulk[buf][threadIdx.x][0]);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(NQ * 16) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst), "l"(src), "r"(NQ * 16), "r"(bar) : "memory");
            } else {
#pragma unroll
                for (int q = 0; q < NQ; q++) {
                    uint32_t dst = (uint32_t)__cvta_generic_to_shared(&s_pts[buf][q][threadIdx.x]);
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + 16 * q) : "memory");
                }
            }
        };
        if (len) prefetch(e_next, 0);
        if (!TMA) asm volatile("cp.async.commit_group;" ::: "memory");
        for (uint32_t k = 0; k < len; k++) {
            const uint32_t e = e_next, neg = e >> 31;
            const int buf = k & 1;
            if (k + 1 < len) { e_next = idx[k + 1]; prefetch(e_next, buf ^ 1); }
            uint32_t words[NQ * 4];
            if (TMA) {
                const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&s_bar[buf][threadIdx.x]);
                const uint32_t parity = (k >> 1) & 1u;
                uint32_t done;
                do {
                    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
                } while (!done);
                const uint4 *sp = reinterpret_cast<const uint4 *>(&s_bulk[buf][threadIdx.x][0]);
#pragma unroll
                for (int q = 0; q < NQ; q++) { uint4 v = sp[q]; words[4 * q] = v.x; words[4 * q + 1] = v.y; words[4 * q + 2] = v.z; words[4 * q + 3] = v.w; }
            } else {
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 1;" ::: "memory");
#pragma unroll
                for (int q = 0; q < NQ; q++) { uint4 v = s_pts[buf][q][threadIdx.x]; words[4 * q] = v.x; words[4 * q + 1] = v.y; words[4 * q + 2] = v.z; words[4 * q + 3] = v.w; }
            }
            ge_niels_packed pk;
#pragma unroll
            for (int q = 0; q < 24; q++) pk.w[q] = words[q];
            ge64_niels nl; ge64_niels_unpack(nl, pk);
            ge64_madd(acc64, acc64, nl, neg);
        }
        ge64_to_p3(acc, acc64);
    } else {
    if (fold_old) load_p3(acc, buckets + t); else ge_p3_identity(acc);
    for (uint32_t k = 0; k < len; k++) {
        uint32_t e = idx[k];
        uint32_t neg = e >> 31, pi = e & 0x7fffffffu;
        const uint4 *src = reinterpret_cast<const uint4 *>(reinterpret_cast<const ge_niels_packed *>(points) + pi);
        ge_niels_packed pk;
#pragma unroll
        for (int q = 0; q < 6; q++) { uint4 v = __ldg(src + q); pk.w[4 * q] = v.x; pk.w[4 * q + 1] = v.y; pk.w[4 * q + 2] = v.z; pk.w[4 * q + 3] = v.w; }
        ge_niels nl; ge_niels_unpack(nl, pk);
        ge_madd(acc, acc, nl, neg);
    }
    }
    ge_p3_raw r; ge_p3_store_raw(r, acc);
    uint4 *o = reinterpret_cast<uint4 *>(!split ? buckets + t : task_sums + p);
#pragma unroll
    for (int q = 0; q < 10; q++) o[q] = make_uint4(r.w[4 * q], r.w[4 * q + 1], r.w[4 * q + 2], r.w[4 * q + 3]);
}

// Everything below is latency-bound tree work on few points: k_heavy_fixup and k_plain_sum run on groups of four
// lanes (warp4.cuh), one point operation per group at a time; k_chunk_reduce and k_finish_windows spread the limbs of
// one point over 20 lanes of a warp (warp4_f64.cuh).

// One warp per heavy bucket (grid-stride over the heavy list): the 8 groups of the warp take
// strided task sums, then a 3-level shuffle tree across groups.
__global__ void __launch_bounds__(128)
k_heavy_fixup(const uint32_t *__restrict__ heavy, const uint32_t *__restrict__ ntasks, const uint32_t *__restrict__ task_off,
              const uint32_t *__restrict__ win_base, uint32_t nbuckets, uint32_t w0, uint32_t w1,
              const ge_p3_raw *__restrict__ task_sums, ge_p3_raw *__restrict__ buckets, int first)
{
    const uint32_t lane = threadIdx.x & 31, role = lane & 3, grp = lane >> 2;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t nheavy = heavy[0];
    for (uint32_t h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; h < nheavy; h += nwarps) {
        uint32_t tb = heavy[1 + h];
        if (tb / nbuckets < w0 || tb / nbuckets >= w1) continue;      // another window group's bucket
        uint32_t kk = ntasks[tb];
        uint32_t base = win_base[tb / nbuckets] + task_off[tb];
        w4_point acc, x;
        if (first || grp != 0) w4_identity(acc); else w4_load(acc, buckets + tb);   // later chunks: keep the old sum
        for (uint32_t j0 = 0; j0 < kk; j0 += 8) {          // uniform trip count across the warp
            uint32_t j = j0 + grp;
            if (j < kk) w4_load(x, task_sums + base + j); else w4_identity(x);
            w4_add(acc, x, role);
        }
        for (int d = 16; d >= 4; d >>= 1) { w4_shfl_down(x, acc, d); w4_add(acc, x, role); }
        if (grp == 0) w4_store(buckets + tb, acc, role);
    }
}

__device__ __forceinline__ void load_p3_f64(ge64_p3 &o, const ge_p3_raw *src)
{
    ge_p3 q; load_p3(q, src);
    fe64_from_fe_limbs(o.X, q.X); fe64_from_fe_limbs(o.Y, q.Y); fe64_from_fe_limbs(o.Z, q.Z); fe64_from_fe_limbs(o.T, q.T);
}

// Level 1 of the bucket reduction (see k_chunk_reduce below) with ONE THREAD per chunk of m buckets on the
// FP64-pipe field: 2^(c-1) W / m chunks (32768 for 2^20 pairs) are enough threads for the throughput field, and
// a thread's 2(m-1) additions need no shuffles.  S_q = sum_r B_{qm+r},  W_q = sum_r (r+1) B_{qm+r}.
__global__ void __launch_bounds__(32)
k_chunk_reduce_f64(const ge_p3_raw *__restrict__ S_in, uint32_t n_in, uint32_t m, uint32_t n_out, uint32_t nwin,
                   ge_p3_raw *__restrict__ S_out, ge_p3_raw *__restrict__ W_out)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_out * nwin) return;
    const uint32_t w = t / n_out, q = t % n_out;
    const ge_p3_raw *S = S_in + (size_t)w * n_in + (size_t)q * m;
    fe64 d2; fe64_const_2d(d2);
    ge64_p3 run, acc, x;
    load_p3_f64(run, S + (m - 1));
    acc = run;
    ge_p3 nxt;                                              // the next bucket is loaded one iteration ahead
    if (m > 1) load_p3(nxt, S + (m - 2));
#pragma unroll 1
    for (uint32_t r = m - 1; r-- > 0;) {
        fe64_from_fe_limbs(x.X, nxt.X); fe64_from_fe_limbs(x.Y, nxt.Y); fe64_from_fe_limbs(x.Z, nxt.Z); fe64_from_fe_limbs(x.T, nxt.T);
        if (r > 0) load_p3(nxt, S + (r - 1));
        ge64_add_p3(run, run, x, d2);
        ge64_add_p3(acc, acc, run, d2);
    }
    ge_p3 o; ge_p3_raw raw;
    ge64_to_p3(o, run); ge_p3_store_raw(raw, o);
    uint4 *d = reinterpret_cast<uint4 *>(S_out + t);
#pragma unroll
    for (int k = 0; k < 10; k++) d[k] = make_uint4(raw.w[4 * k], raw.w[4 * k + 1], raw.w[4 * k + 2], raw.w[4 * k + 3]);
    ge64_to_p3(o, acc); ge_p3_store_raw(raw, o);
    d = reinterpret_cast<uint4 *>(W_out + t);
#pragma unroll
    for (int k = 0; k < 10; k++) d[k] = make_uint4(raw.w[4 * k], raw.w[4 * k + 1], raw.w[4 * k + 2], raw.w[4 * k + 3]);
}

// Bucket reduction  sum_b (b+1) B_b  per window (pippenger.rs:146-151), in log depth:
//   level 1   chunks of m buckets: S_q = sum_r B_{qm+r},  W_q = sum_r (r+1) B_{qm+r}   (running sums)
//   level l   chunks of m items of S^{l-1}: S^l_q, W^l_q = sum_r r S^{l-1}_{qm+r}      (0-based weights)
//   then      target = A_1 + m_1 (A_2 + m_2 (A_3 + ...)),  A_l = plain sum of the W^l array
// Doublings happen once per level in the final per-window Horner, not inside every level.
// One warp per chunk, the limbs of each point spread over 20 lanes (warp4_f64.cuh); n_in is a power of two and m
// divides it, so every chunk has m items.
__global__ void __launch_bounds__(128)
k_chunk_reduce(const ge_p3_raw *__restrict__ S_in, uint32_t n_in, uint32_t m, uint32_t one_based, uint32_t n_out,
               uint32_t nwin, ge_p3_raw *__restrict__ S_out, ge_p3_raw *__restrict__ W_out)
{
    const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= n_out * nwin) return;                                                  // whole warps
    const w20_role rl = w20_roles();
    const double d2 = w20_const_2d(rl);
    const uint32_t w = t / n_out, q = t % n_out;
    const ge_p3_raw *S = S_in + (size_t)w * n_in + (size_t)q * m;
    double run = w20_load(S + (m - 1), rl), acc = run;
#pragma unroll 1
    for (uint32_t r = m - 1; r-- > 1;) {
        w20_add(run, w20_load(S + r, rl), d2, rl);
        w20_add(acc, run, d2, rl);
    }
    if (m > 1) {
        w20_add(run, w20_load(S, rl), d2, rl);
        if (one_based) w20_add(acc, run, d2, rl);
    } else if (!one_based) {
        acc = w20_identity(rl);
    }
    w20_store(S_out + t, run);
    w20_store(W_out + t, acc);
}

// plain sum of one array per CTA (blockIdx.x = array id): 32 groups take strided items, then a
// shared-memory tree over the 32 partial sums
// Arrays are described by (offset, length) pairs in device memory (fixed per window width, cached in the
// context).  Two stages: pieces of at most SUM_PIECE items, then the per-array sum of the piece sums.
#define SUM_PIECE 256u
__global__ void __launch_bounds__(128)
k_plain_sum(const ge_p3_raw *__restrict__ pool, const uint2 *__restrict__ desc, ge_p3_raw *__restrict__ out)
{
    __shared__ ge_p3_raw sh[32];
    const uint32_t role = threadIdx.x & 3, grp = threadIdx.x >> 2;
    const uint2 d = desc[blockIdx.x];
    const ge_p3_raw *a = pool + d.x;
    const uint32_t len = d.y;
    w4_point acc, x;
    w4_identity(acc);
    for (uint32_t i0 = 0; i0 < len; i0 += 32) {
        uint32_t i = i0 + grp;
        if (i < len) w4_load(x, a + i); else w4_identity(x);
        w4_add(acc, x, role);
    }
    w4_store(&sh[grp], acc, role);
    __syncthreads();
    for (uint32_t d = 16; d > 0; d >>= 1) {
        if (threadIdx.x < 32 * ((d + 7) / 8)) {            // whole warps only
            uint32_t g2 = grp < d ? grp + d : grp;        // idle groups add their own value (discarded)
            w4_load(acc, &sh[grp]); w4_load(x, &sh[g2]);
            w4_add(acc, x, role);
        }
        __syncthreads();
        if (grp < d) w4_store(&sh[grp], acc, role);
        __syncthreads();
    }
    if (grp == 0) { w4_load(acc, &sh[0]); w4_store(out + blockIdx.x, acc, role); }
}

// per window: target = A_1 + m_1 (A_2 + m_2 (...)); A sums are laid out [level][window]
struct LevelInfo { int nlevels; int log2m[16]; };
__global__ void __launch_bounds__(128)
k_finish_windows(const ge_p3_raw *__restrict__ S_top, const ge_p3_raw *__restrict__ A, LevelInfo li, uint32_t nwin,
                 ge_p3_raw *__restrict__ out)
{
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;               // one warp per window, 20 lanes
    if (w >= nwin) return;
    const w20_role rl = w20_roles();
    double t;
    if (li.nlevels > 0) {
        const double d2 = w20_const_2d(rl);
        t = w20_load(A + (size_t)(li.nlevels - 1) * nwin + w, rl);
#pragma unroll 1
        for (int l = li.nlevels - 2; l >= 0; l--) {
#pragma unroll 1
            for (int k = 0; k < li.log2m[l]; k++) w20_dbl(t, rl);
            w20_add(t, w20_load(A + (size_t)l * nwin + w, rl), d2, rl);
        }
    } else {
        t = w20_load(S_top + w, rl);      // a single bucket of weight 1
    }
    w20_store(out + w, t);
}

// Final Horner over windows (pippenger.rs:159): total = total * 2^c + window, ~250 sequential doublings with the
// limbs of the total spread over 20 lanes (warp4_f64.cuh), then the encoding's inversion on the same lanes.
__global__ void __launch_bounds__(32)
k_combine(const ge_p3_raw *__restrict__ windows, int ranks, int nwin, int c, MsmResult *__restrict__ res)
{
    const w20_role r = w20_roles();
    uint32_t s[8];
    ge_p3 total;
    w20_encode(s, total, w20_horner(windows, ranks, nwin, c, r), r);
    if (threadIdx.x != 0) return;
#pragma unroll
    for (int i = 0; i < 8; i++) res->compressed[i] = s[i];
    fe_to_limbs51(res->limbs, total.X); fe_to_limbs51(res->limbs + 5, total.Y);
    fe_to_limbs51(res->limbs + 10, total.Z); fe_to_limbs51(res->limbs + 15, total.T);
    res->is_identity = ge_is_identity(total);
    res->pad = 0;
}

// Fine bits F of the digit sort: as few coarse bins per window as keep their mean size on uniform digits near
// SORT_BIN_MEAN (half of what k_sort_fine holds in shared memory), within the shared histograms' sizes.
// c = 16, 2^20 pairs: F = 7, 256 coarse bins of 128 buckets per window.
static int msm_sort_fine_bits(size_t entries_per_window, int c, int hist_windows)
{
    int lg = std::max(0, c - 1 - SORT_FINE_MAX);            // log2 of the coarse bins per window
    while (lg < c - 1 && ((size_t)SORT_BIN_MEAN << lg) < entries_per_window && (2u << lg) <= SORT_NC_MAX &&
           ((size_t)hist_windows << (lg + 1)) <= SORT_HIST_MAX)
        lg++;
    return c - 1 - lg;
}

// ------------------------------------------------------------------------------------------
// One chunk of (scalar, point) pairs: digits, counting sort, task lists and bucket accumulation.
// `first` chunks start the buckets at the identity; later chunks add onto them.  All chunks of one
// MSM must use the same window width c.
// `active_windows` > 0 promises that every scalar of this chunk is below 2^(c * active_windows - 1): digits are
// extracted, sorted and accumulated for the low `active_windows` windows only (verify_batch: the 128-bit z_i).
// `flat` (a table stride): d_points holds nwin tables of `flat` points, table w = 2^(cw) P_i (precomp.cu); every digit then goes into ONE
// bucket window, so the reduction handles 2^(c-1) buckets instead of nwin times as many and no doubling is left
// (pair with msm_reduce_finish(..., flat = true)).
int msm_accumulate_chunk(dalek_b200_ctx *ctx, const uint32_t *d_scalars, const ge_niels_packed *d_points, size_t n,
                         int c, bool first, int active_windows, size_t flat, cudaEvent_t points_ready)
{
    const int nwin_d = msm_window_count_for_bits(c);               // digit windows
    const int nact = active_windows > 0 && active_windows < nwin_d ? active_windows : nwin_d;
    const int nwin = flat ? 1 : nwin_d;                            // bucket windows
    const uint32_t nb = 1u << (c - 1);
    const size_t total_buckets = (size_t)nwin * nb;
    const uint32_t task_len = flat ? msm_task_len(n * (size_t)nact, 1, nb) : msm_task_len(n, nact, nb);
    const size_t max_tasks = total_buckets + (std::max<size_t>(1, n) * nact) / task_len + 1;
    const size_t max_heavy = (std::max<size_t>(1, n) * nact) / task_len + 1;
    const uint32_t parts = (nb + SCAN_PART - 1) / SCAN_PART;
    const int F = msm_sort_fine_bits(flat ? n * (size_t)nact : n, c, flat ? 1 : nact);
    const uint32_t nc = nb >> F;                                  // coarse bins per bucket window
    cudaStream_t st = ctx->stream;
    int rc;
    // counts | coarse counts | heavy list (count + entries): one memset clears the coarse counts and the heavy count
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_COUNTS], (total_buckets + (size_t)nwin * nc + 1 + max_heavy) * 4))) return rc;
    // offsets | scan part sums | coarse bin cursors | extra-slice prefix of the bins | extra slices per window
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_OFFSETS], (total_buckets + (size_t)nwin * parts + 2 * (size_t)nwin * nc + nwin) * 4))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_NTASKS], total_buckets * 4))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_TASK_OFF], total_buckets * 4 + (nwin + 1) * 4))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_TASKS], max_tasks * 8))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_TASK_SUMS], max_tasks * sizeof(ge_p3_raw)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_TASK_ORDER], (3 * TASK_BINS + max_tasks) * 4))) return rc;   // hist | cursor | start | order
    // the sort's records: 8 B per non-zero digit, in (bucket window, coarse bin) order
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_DIGITS], std::max<size_t>(1, n) * nact * 8))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_SORTED], std::max<size_t>(1, n) * nact * 4))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_BUCKETS], total_buckets * sizeof(ge_p3_raw)))) return rc;
    uint32_t *counts = (uint32_t *)ctx->ws[WS_MSM_COUNTS].p, *offsets = (uint32_t *)ctx->ws[WS_MSM_OFFSETS].p;
    uint32_t *ntasks = (uint32_t *)ctx->ws[WS_MSM_NTASKS].p, *task_off = (uint32_t *)ctx->ws[WS_MSM_TASK_OFF].p;
    uint32_t *win_base = task_off + total_buckets;
    uint32_t *ccount = counts + total_buckets, *heavy = ccount + (size_t)nwin * nc;
    uint32_t *part_sums = offsets + total_buckets, *ccursor = part_sums + (size_t)nwin * parts;
    uint32_t *xpre = ccursor + (size_t)nwin * nc, *xtot = xpre + (size_t)nwin * nc;
    uint2 *tasks = (uint2 *)ctx->ws[WS_MSM_TASKS].p;
    uint32_t *t_hist = (uint32_t *)ctx->ws[WS_MSM_TASK_ORDER].p, *t_cursor = t_hist + TASK_BINS, *t_start = t_cursor + TASK_BINS;
    uint32_t *order = t_start + TASK_BINS;
    ge_p3_raw *task_sums = (ge_p3_raw *)ctx->ws[WS_MSM_TASK_SUMS].p;
    uint2 *records = (uint2 *)ctx->ws[WS_MSM_DIGITS].p;
    uint32_t *sorted = (uint32_t *)ctx->ws[WS_MSM_SORTED].p;
    ge_p3_raw *buckets = (ge_p3_raw *)ctx->ws[WS_MSM_BUCKETS].p;

    const size_t part_smem = SORT_TILE * 8 + (2 * (size_t)nc + 33) * 4;
    const size_t fine_smem = SORT_FINE_CAP * 12 + ((1u << F) + 33) * 4;
    if (part_smem > SORT_PART_SMEM_MAX || fine_smem > SORT_FINE_SMEM_MAX) {   // msm_sort_fine_bits keeps nc and F in bounds
        ctx->last_error = "msm_accumulate_chunk: digit sort needs more shared memory than its bound";
        return DALEK_E_CUDA;
    }
    if (!ctx->sort_attr_set) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(k_sort_partition, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_PART_SMEM_MAX));
        CUDA_TRY(ctx, cudaFuncSetAttribute(k_sort_fine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_FINE_SMEM_MAX));
        ctx->sort_attr_set = true;
    }
    CUDA_TRY(ctx, cudaMemsetAsync(ccount, 0, ((size_t)nwin * nc + 1) * 4, st));
    CUDA_TRY(ctx, cudaMemsetAsync(t_hist, 0, 2 * TASK_BINS * 4, st));
    if (n) {
        k_sort_count<<<cdiv(n, SORT_COUNT_TILE), SORT_THREADS, 0, st>>>((const uint4 *)d_scalars, n, c, nact, F, nc, flat ? 1 : 0, ccount);
        ctx->launches++;
    }
    // ntasks is free until k_task_count: it holds the fill counters of the big bins' buckets
    k_sort_bins_scan<<<nwin, SORT_THREADS, 0, st>>>(ccount, nc, F, nb, ccursor, xpre, xtot, counts, ntasks);
    if (n) {
        k_sort_partition<<<cdiv(n, SORT_TILE), SORT_THREADS, part_smem, st>>>((const uint4 *)d_scalars, n, c, nact, F, nc, nb, flat,
                                                                              ccount, ccursor, records, counts);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());     // a lost sort launch leaves records unwritten: enqueue nothing that reads them
    }
    const size_t extra = n * (size_t)nact / SORT_FINE_CAP;          // bounds the extra slices of all big bins
    k_sort_fine<<<(unsigned)(nwin * nc + extra), SORT_THREADS, fine_smem, st>>>(records, ccount, ccursor, xpre, xtot, n, F, nc, nb,
                                                                               (uint32_t)nwin, flat ? 1 : 0, counts, offsets, sorted, ntasks);
    CUDA_TRY(ctx, cudaGetLastError());
    k_task_count<<<cdiv(total_buckets, 256), 256, 0, st>>>(counts, (uint32_t)total_buckets, task_len, ntasks, heavy);
    k_scan_partial<<<nwin * parts, 1024, 0, st>>>(ntasks, nb, parts, part_sums);
    k_scan_bases<<<nwin, 32, 0, st>>>(part_sums, parts);
    k_scan_apply<<<nwin * parts, 1024, 0, st>>>(ntasks, part_sums, nb, parts, task_off);
    k_task_bases<<<1, 32, 0, st>>>(ntasks, task_off, nb, nwin, win_base);
    k_task_fill<<<cdiv(total_buckets, 256), 256, 0, st>>>(ntasks, task_off, win_base, nb, (uint32_t)total_buckets, tasks);
    k_task_hist<<<cdiv(max_tasks, 256), 256, 0, st>>>(tasks, counts, win_base + nwin, task_len, t_hist);
    k_task_scan<<<1, 256, 0, st>>>(t_hist, t_start);
    k_task_scatter<<<cdiv(max_tasks, 256), 256, 0, st>>>(tasks, counts, win_base + nwin, task_len, t_start, t_cursor, order);
    ctx->launches += 11;
    // the digit / sort passes above only read the scalars: the conversion of the points may still be running on another stream
    if (points_ready) CUDA_TRY(ctx, cudaStreamWaitEvent(st, points_ready, 0));
    if (first) CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    {
        const unsigned grid = cdiv(max_tasks, 128);
        const int f = first ? 1 : 0;
#define LAUNCH_ACC(F64_, TMA_) k_bucket_accumulate<F64_, TMA_><<<grid, 128, 0, st>>>(d_points, sorted, counts, offsets, ntasks, tasks, order, win_base, 0, nwin, n, nb, task_len, buckets, task_sums, f)
        const bool tma = ctx->opt_field_f64 && ctx->opt_acc_tma;
        if (tma) LAUNCH_ACC(1, 1); else if (ctx->opt_field_f64) LAUNCH_ACC(1, 0); else LAUNCH_ACC(0, 0);
#undef LAUNCH_ACC
        k_heavy_fixup<<<ctx->sm_count * 4, 128, 0, st>>>(heavy, ntasks, task_off, win_base, nb, 0u, (uint32_t)nwin, task_sums, buckets, f);
        ctx->launches += 2;
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));          // ev_a .. ev_b brackets the accumulation kernels
    ctx->last_kernel_launches = first ? 1 : ctx->last_kernel_launches + 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

// Bucket reduction of all windows, and (if d_result) the Horner over windows + encoding.
// flat: the buckets are the single window filled by msm_accumulate_chunk(..., flat = true): d_windows[0] is already
// the whole sum and d_result (if given) needs no doubling.
int msm_reduce_finish(dalek_b200_ctx *ctx, int c, ge_p3_raw *d_windows, MsmResult *d_result, bool flat)
{
    const int nwin = flat ? 1 : msm_window_count_for_bits(c);
    const int desc_key = c + (flat ? 64 : 0);
    const uint32_t nb = 1u << (c - 1);
    cudaStream_t st = ctx->stream;
    int rc;
    ge_p3_raw *buckets = (ge_p3_raw *)ctx->ws[WS_MSM_BUCKETS].p;
    LevelInfo li; li.nlevels = 0;
    std::vector<uint32_t> lvl_m, lvl_nout;
    size_t pool_pts = 0;
    {
        uint32_t n_in = nb; bool first = true;
        while (n_in > 1) {
            uint32_t m = first ? std::min<uint32_t>(n_in, 16) : std::min<uint32_t>(n_in, 8);
            uint32_t n_out = (n_in + m - 1) / m;
            lvl_m.push_back(m); lvl_nout.push_back(n_out);
            int lg = 0; while ((1u << lg) < m) lg++;
            li.log2m[li.nlevels++] = lg;
            pool_pts += 2 * (size_t)n_out * nwin;
            n_in = n_out; first = false;
        }
    }
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_REDUCE_POOL], std::max<size_t>(1, pool_pts) * sizeof(ge_p3_raw)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_REDUCE_SUMS], (size_t)16 * nwin * sizeof(ge_p3_raw)))) return rc;
    ge_p3_raw *pool = (ge_p3_raw *)ctx->ws[WS_MSM_REDUCE_POOL].p, *A = (ge_p3_raw *)ctx->ws[WS_MSM_REDUCE_SUMS].p;
    const ge_p3_raw *S_in = buckets;
    uint32_t n_in = nb;
    size_t pos = 0;
    std::vector<std::pair<size_t, uint32_t>> w_arrays;        // (offset of W array, n_out) per level
    for (int l = 0; l < li.nlevels; l++) {
        uint32_t m = lvl_m[l], n_out = lvl_nout[l];
        ge_p3_raw *S_out = pool + pos, *W_out = pool + pos + (size_t)n_out * nwin;
        if (l == 0 && ctx->opt_field_f64 && n_in % m == 0)
            k_chunk_reduce_f64<<<cdiv((size_t)n_out * nwin, 32), 32, 0, st>>>(S_in, n_in, m, n_out, nwin, S_out, W_out);   // small CTAs: 1024 warps spread evenly over the SMs
        else
            k_chunk_reduce<<<cdiv((size_t)n_out * nwin * 32, 128), 128, 0, st>>>(S_in, n_in, m, l == 0 ? 1u : 0u, n_out, nwin, S_out, W_out);
        ctx->launches++;
        w_arrays.push_back({pos + (size_t)n_out * nwin, n_out});
        S_in = S_out; n_in = n_out; pos += 2 * (size_t)n_out * nwin;
    }
    {   // plain sums of every (level, window) W array, two stages; descriptors depend only on c
        std::vector<uint2> d1, d2;
        for (int l = 0; l < li.nlevels; l++)
            for (int w = 0; w < nwin; w++) {
                uint32_t off = (uint32_t)(w_arrays[l].first + (size_t)w * w_arrays[l].second), len = w_arrays[l].second;
                uint32_t first_piece = (uint32_t)d1.size();
                for (uint32_t o = 0; o < len; o += SUM_PIECE) d1.push_back(make_uint2(off + o, std::min(SUM_PIECE, len - o)));
                d2.push_back(make_uint2(first_piece, (uint32_t)d1.size() - first_piece));
            }
        const size_t n1 = d1.size(), n2 = d2.size();
        if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_SUM_DESC], (n1 + n2) * sizeof(uint2)))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_SUM_PART], n1 * sizeof(ge_p3_raw)))) return rc;
        uint2 *dd1 = (uint2 *)ctx->ws[WS_MSM_SUM_DESC].p, *dd2 = dd1 + n1;
        if (ctx->sum_desc_c != desc_key) {
            CUDA_TRY(ctx, cudaMemcpyAsync(dd1, d1.data(), n1 * sizeof(uint2), cudaMemcpyHostToDevice, st));
            CUDA_TRY(ctx, cudaMemcpyAsync(dd2, d2.data(), n2 * sizeof(uint2), cudaMemcpyHostToDevice, st));
            CUDA_TRY(ctx, cudaStreamSynchronize(st));       // d1/d2 are host temporaries (rare: once per width)
            ctx->sum_desc_c = desc_key;
        }
        ge_p3_raw *parts = (ge_p3_raw *)ctx->ws[WS_MSM_SUM_PART].p;
        k_plain_sum<<<(unsigned)n1, 128, 0, st>>>(pool, dd1, parts);
        k_plain_sum<<<(unsigned)n2, 128, 0, st>>>(parts, dd2, A);
        ctx->launches += 2;
    }
    k_finish_windows<<<cdiv((size_t)nwin * 32, 128), 128, 0, st>>>(S_in, A, li, nwin, d_windows);
    ctx->launches++;
    if (d_result) {
        k_combine<<<1, 32, 0, st>>>(d_windows, 1, nwin, c, d_result);
        ctx->launches++;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

int msm_combine_windows(dalek_b200_ctx *ctx, const ge_p3_raw *d_windows, int ranks, int nwin, int c, MsmResult *d_result)
{
    k_combine<<<1, 32, 0, ctx->stream>>>(d_windows, ranks, nwin, c, d_result);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}
