// precomp.cu -- VartimePrecomputedMultiscalarMul (curve25519-dalek/src/traits.rs:290-406) for EdwardsPoint and
// RistrettoPoint (VartimeEdwardsPrecomputation, src/edwards.rs:1038-1076; VartimeRistrettoPrecomputation,
// src/ristretto.rs:1004-1049; serial backend precomputed_straus.rs:33-127).
//
// The reference precomputes width-8 NAF tables of the static points so that repeated calls skip that work.
// Here the precomputation is what the bucket MSM can reuse between calls, RESIDENT in HBM:
//   * the static points decoded and converted to packed affine Niels form (96 B each, what the bucket kernel reads), and
//   * with the option "precomp_tables" and >= 4096 points, the tables 2^(c w) P_i for every window w of the width c
//     chosen at construction, as affine Niels points (96 B each, 1.7 GB for 2^20 points at c = 16).  With them a
//     digit of window w selects from table w and ALL windows share one set of 2^(c-1) buckets: the reduction shrinks
//     by the window count and the final Horner (256 sequential doublings) disappears.  But the bucket kernel then gathers from 1.7 GB at random instead of from the 128 MB point
//     array, and that costs it most of what the tail saves (tools/sweep_precomp.py times both).  Hence off by default.
// A call moves only scalars (32 B per static point instead of 192 B).  Dynamic terms go through the ordinary
// multi-window path and the two partial results are added.  The result is the same group element as the
// reference's (tests compare canonical encodings).
#include <algorithm>
#include <cstring>
#include <new>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "ge64.cuh"

struct dalek_b200_precomp {
    dalek_b200_ctx *ctx;
    ge_niels_packed *d_points;  // n packed affine Niels points, device
    int ristretto;         // 1: inputs/outputs are Ristretto encodings
    size_t n;
    ge_niels_packed *d_table;   // nwin slabs of n affine Niels points: slab w holds 2^(c w) P_i; null if not built
    int c, nwin;
};

// P_i from the packed affine Niels form (y+x, y-x, 2dxy): x = ((y+x) - (y-x)) / 2, y = ((y+x) + (y-x)) / 2
__device__ __forceinline__ void point_from_packed(ge_p3 &p, const ge_niels_packed *packed, size_t i)
{
    fe ypx, ymx, half, t;
    ge_niels_packed q = packed[i];
    fe_frombytes_words(ypx, q.w); fe_frombytes_words(ymx, q.w + 8);
    const uint32_t half_words[8] = {0xfffffff7u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
    fe_frombytes_words(half, half_words);                 // (p + 1) / 2 = 2^254 - 9
    fe_sub(t, ypx, ymx); fe_mul(p.X, t, half);
    fe_add(t, ypx, ymx); fe_mul(p.Y, t, half);
    fe_1(p.Z);
    fe_mul(p.T, p.X, p.Y);
}

__global__ void __launch_bounds__(128, 2)
k_precomp_table(const ge_niels_packed *__restrict__ packed, size_t n, int c, int nwin, ge_niels_packed *__restrict__ table)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 P;
    point_from_packed(P, packed, i);
    ge64_p3 Q; ge64_from_p3(Q, P);
#pragma unroll 1
    for (int w = 0; w < nwin; w++) {
        ge_p3 A; ge64_to_p3(A, Q);
        fe zi, x, y;
        fe_invert_f64(zi, A.Z);
        fe_mul(x, A.X, zi); fe_mul(y, A.Y, zi);
        ge_niels nl; ge_affine_to_niels(nl, x, y);
        ge_niels_packed pk; ge_niels_pack(pk, nl);
        uint4 *o = reinterpret_cast<uint4 *>(table + (size_t)w * n + i);
#pragma unroll
        for (int k = 0; k < 6; k++) o[k] = make_uint4(pk.w[4 * k], pk.w[4 * k + 1], pk.w[4 * k + 2], pk.w[4 * k + 3]);
        if (w + 1 < nwin)
#pragma unroll 1
            for (int k = 0; k < c; k++) ge64_dbl(Q, Q);
    }
}

// R = R1 + R2 of two MSM results (limbs), re-encoded
__global__ void k_add_results(const MsmResult *__restrict__ a, const MsmResult *__restrict__ b, MsmResult *__restrict__ out)
{
    ge_p3 p, q, r;
    fe_from_limbs51(p.X, a->limbs); fe_from_limbs51(p.Y, a->limbs + 5); fe_from_limbs51(p.Z, a->limbs + 10); fe_from_limbs51(p.T, a->limbs + 15);
    fe_from_limbs51(q.X, b->limbs); fe_from_limbs51(q.Y, b->limbs + 5); fe_from_limbs51(q.Z, b->limbs + 10); fe_from_limbs51(q.T, b->limbs + 15);
    ge_add(r, p, q);
    uint32_t s[8];
    ge_compress(s, r);
    for (int k = 0; k < 8; k++) out->compressed[k] = s[k];
    fe_to_limbs51(out->limbs, r.X); fe_to_limbs51(out->limbs + 5, r.Y); fe_to_limbs51(out->limbs + 10, r.Z); fe_to_limbs51(out->limbs + 15, r.T);
    out->is_identity = ge_is_identity(r);
    out->pad = 0;
}

extern "C" {

int dalek_b200_precomp_new(dalek_b200_ctx *ctx, const void *static_points, int point_fmt, size_t n, dalek_b200_precomp **out)
{
    if (!ctx || !out || (n && !static_points) || n >= (1ull << 31) ||
        (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED && point_fmt != DALEK_POINTS_RISTRETTO))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    dalek_b200_precomp *pre = new (std::nothrow) dalek_b200_precomp();
    if (!pre) return DALEK_E_NOMEM;
    pre->ctx = ctx; pre->n = n; pre->ristretto = point_fmt == DALEK_POINTS_RISTRETTO;
    pre->d_points = nullptr;
    if (cudaMalloc((void **)&pre->d_points, std::max<size_t>(1, n) * sizeof(ge_niels_packed)) != cudaSuccess) {
        ctx->last_error = "cudaMalloc failed for the static point table";
        delete pre;
        return DALEK_E_NOMEM;
    }
    auto fail = [&](int code) { cudaFree(pre->d_points); delete pre; return code; };
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * msm_point_bytes(point_fmt)))) return fail(rc);
    if ((rc = msm_driver_ws_reserve(ctx))) return fail(rc);
    if ((rc = pinned_reserve(ctx, 256))) return fail(rc);
    int *h_bad = (int *)ctx->h_pinned;
    *h_bad = 0;
    if (cudaMemsetAsync(ctx->ws[WS_FLAGS].p, 0, FLAG_WORDS * sizeof(int), st) != cudaSuccess) return fail(DALEK_E_CUDA);
    if (n && cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, static_points, n * msm_point_bytes(point_fmt), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return fail(DALEK_E_CUDA);
    if ((rc = msm_prepare_points(ctx, ctx->ws[WS_STAGING_IN].p, point_fmt, n, pre->d_points, (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS))) return fail(rc);
    if (cudaMemcpyAsync(h_bad, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(DALEK_E_CUDA);
    if (cudaStreamSynchronize(st) != cudaSuccess) return fail(DALEK_E_CUDA);
    if (*h_bad) { ctx->last_error = "a static point does not decode"; return fail(DALEK_NONE); }
    pre->d_table = nullptr; pre->c = 0; pre->nwin = 0;
    if (ctx->opt_precomp_tables && n >= 4096) {
        pre->c = msm_choose_window_bits(ctx, n);
        pre->nwin = msm_window_count_for_bits(pre->c);
        const size_t bytes = (size_t)pre->nwin * n * sizeof(ge_niels_packed);
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && bytes < free_b / 2 && (size_t)pre->nwin * n < (1ull << 31) &&
            cudaMalloc((void **)&pre->d_table, bytes) == cudaSuccess) {
            k_precomp_table<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(pre->d_points, n, pre->c, pre->nwin, pre->d_table);
            ctx->launches++;
            if (cudaStreamSynchronize(st) != cudaSuccess) { cudaFree(pre->d_table); return fail(DALEK_E_CUDA); }
        } else {
            pre->d_table = nullptr;                          // not enough memory: the resident points alone still serve
            (void)cudaGetLastError();
        }
    }
    *out = pre;
    return DALEK_OK;
}

size_t dalek_b200_precomp_len(const dalek_b200_precomp *pre) { return pre ? pre->n : 0; }

void dalek_b200_precomp_destroy(dalek_b200_precomp *pre)
{
    if (!pre) return;
    cudaSetDevice(pre->ctx->device);
    cudaStreamSynchronize(pre->ctx->stream);
    if (pre->d_points) cudaFree(pre->d_points);
    if (pre->d_table) cudaFree(pre->d_table);
    delete pre;
}

int dalek_b200_precomp_mixed_msm(dalek_b200_ctx *ctx, const dalek_b200_precomp *pre, const uint8_t *static_scalars, size_t n_static,
                                 const uint8_t *dynamic_scalars, const void *dynamic_points, int dynamic_fmt, size_t n_dynamic,
                                 uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!ctx || !pre || pre->ctx != ctx || (n_static && !static_scalars) || (n_dynamic && (!dynamic_scalars || !dynamic_points)))
        return DALEK_E_INVALID_ARG;
    if (n_static > pre->n) { ctx->last_error = "more static scalars than static points (traits.rs:317-319)"; return DALEK_E_INVALID_ARG; }
    if (dynamic_fmt != DALEK_POINTS_COMPRESSED && dynamic_fmt != DALEK_POINTS_EXTENDED && dynamic_fmt != DALEK_POINTS_RISTRETTO)
        return DALEK_E_INVALID_ARG;
    if (n_dynamic && (dynamic_fmt == DALEK_POINTS_RISTRETTO) != (pre->ristretto != 0) && dynamic_fmt != DALEK_POINTS_EXTENDED)
        return DALEK_E_INVALID_ARG;                     // Edwards and Ristretto encodings do not mix
    if (n_static + n_dynamic >= (1ull << 31)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    cudaStream_t st = ctx->stream;
    const size_t din = msm_point_bytes(dynamic_fmt);
    const bool use_table = pre->d_table != nullptr && n_static > 0;
    // window widths: the table fixes the static width; the dynamic part picks its own
    const int c = use_table ? pre->c : msm_choose_window_bits(ctx, n_static + n_dynamic);
    const int c_dyn = use_table ? msm_choose_window_bits(ctx, n_dynamic) : c;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n_static + n_dynamic) * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n_dynamic) * din))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], std::max<size_t>(1, n_dynamic) * sizeof(ge_niels_packed)))) return rc;
    ge_niels_packed *d_dpts = (ge_niels_packed *)ctx->ws[WS_STAGING_OUT].p;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_FLAGS].p, 0, FLAG_WORDS * sizeof(int), st));
    uint32_t *d_ss = (uint32_t *)ctx->ws[WS_SCALARS].p, *d_ds = d_ss + 8 * n_static;
    MsmResult *d_res = (MsmResult *)ctx->ws[WS_MSM_RESULT].p, *d_r1 = d_res + 1, *d_r2 = d_res + 2;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream_copy, ctx->ev_fork, 0));
    // static scalars in up to 4 chunks, then the dynamic inputs, all on the copy stream
    const int K = n_static >= (1u << 18) ? (int)std::min<long>(4, std::max<long>(1, ctx->opt_host_chunks)) : 1;
    for (int k = 0; k < K; k++) {
        const size_t i0 = n_static * k / K, i1 = n_static * (k + 1) / K;
        if (i1 > i0) CUDA_TRY(ctx, cudaMemcpyAsync(d_ss + 8 * i0, static_scalars + 32 * i0, (i1 - i0) * 32, cudaMemcpyHostToDevice, ctx->stream_copy));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_grp[k], ctx->stream_copy));
    }
    if (n_dynamic) {
        CUDA_TRY(ctx, cudaMemcpyAsync(d_ds, dynamic_scalars, n_dynamic * 32, cudaMemcpyHostToDevice, ctx->stream_copy));
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, dynamic_points, n_dynamic * din, cudaMemcpyHostToDevice, ctx->stream_copy));
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_grp[K], ctx->stream_copy));
    for (int k = 0; k < K; k++) {
        const size_t i0 = n_static * k / K, i1 = n_static * (k + 1) / K;
        CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_grp[k], 0));
        if (use_table) {
            // one bucket window: the digit of window w of scalar i selects table[w * n + i]
            if ((rc = msm_accumulate_chunk(ctx, d_ss + 8 * i0, pre->d_table + i0, i1 - i0, c, k == 0, 0, pre->n))) return rc;
        } else {
            if ((rc = msm_accumulate_chunk(ctx, d_ss + 8 * i0, pre->d_points + i0, i1 - i0, c, k == 0))) return rc;
        }
    }
    CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_grp[K], 0));
    if (use_table) {
        if ((rc = msm_reduce_finish(ctx, c, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, n_dynamic ? d_r1 : d_res, true))) return rc;
        if (n_dynamic) {
            if ((rc = msm_prepare_points(ctx, ctx->ws[WS_STAGING_IN].p, dynamic_fmt, n_dynamic, d_dpts, (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS))) return rc;
            if ((rc = msm_accumulate_chunk(ctx, d_ds, d_dpts, n_dynamic, c_dyn, true))) return rc;
            if ((rc = msm_reduce_finish(ctx, c_dyn, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, d_r2))) return rc;
            k_add_results<<<1, 1, 0, st>>>(d_r1, d_r2, d_res);
            ctx->launches++;
        }
    } else {
        if (n_dynamic) {
            if ((rc = msm_prepare_points(ctx, ctx->ws[WS_STAGING_IN].p, dynamic_fmt, n_dynamic, d_dpts, (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS))) return rc;
            if ((rc = msm_accumulate_chunk(ctx, d_ds, d_dpts, n_dynamic, c, false))) return rc;
        }
        if ((rc = msm_reduce_finish(ctx, c, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, d_res))) return rc;
    }
    uint32_t *d_enc = pre->ristretto ? (uint32_t *)(d_res + 3) : nullptr;
    if (d_enc && (rc = ristretto_encode_result(ctx, d_res, d_enc))) return rc;
    // DALEK_NONE: a dynamic point was None (optional_mixed_multiscalar_mul)
    return msm_read_result(ctx, d_res, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS, d_enc, out_compressed, out_limbs);
}

}  // extern "C"
