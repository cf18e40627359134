// api.cu -- the extern "C" boundary of libdalek_b200.so (include/dalek_b200.h): context handling,
// host<->device staging and the vartime MSM entry points (Edwards and Ristretto).  verify_batch lives in batch.cu, the
// constant-time MSM and the Ristretto double-base batch in straus.cu.
#include <cstring>
#include <new>
#include <random>

#include "../../include/dalek_b200.h"
#include "engine.h"

extern "C" {

int dalek_b200_init(int device, dalek_b200_ctx **out)
{
    if (!out) return DALEK_E_INVALID_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return DALEK_E_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return DALEK_E_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return DALEK_E_NO_DEVICE;   // built for sm_90a only; no fallback path
    if (cudaSetDevice(device) != cudaSuccess) return DALEK_E_CUDA;
    dalek_b200_ctx *ctx = new (std::nothrow) dalek_b200_ctx();
    if (!ctx) return DALEK_E_NOMEM;
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    try { std::random_device rd; for (int i = 0; i < 4; i++) ctx->hash_seed[i] ^= rd(); } catch (...) { }   // results never depend on it
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);       // (greatest priority is the lower number)
    if (cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, prio_lo) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->stream_copy, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->stream3, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->stream_hash, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaEventCreate(&ctx->ev_a) != cudaSuccess || cudaEventCreate(&ctx->ev_b) != cudaSuccess ||
        cudaEventCreate(&ctx->ev_call0) != cudaSuccess || cudaEventCreate(&ctx->ev_call1) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_join2, cudaEventDisableTiming) != cudaSuccess) {
        delete ctx;
        return DALEK_E_CUDA;
    }
    for (int i = 0; i < 8; i++)
        if (cudaEventCreateWithFlags(&ctx->ev_grp[i], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&ctx->ev_hram[i], cudaEventDisableTiming) != cudaSuccess || cudaEventCreate(&ctx->ev_prep[i][0]) != cudaSuccess ||
            cudaEventCreate(&ctx->ev_prep[i][1]) != cudaSuccess) { delete ctx; return DALEK_E_CUDA; }
    *out = ctx;
    return DALEK_OK;
}

void dalek_b200_destroy(dalek_b200_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->stream2);
    cudaStreamSynchronize(ctx->stream3);
    cudaStreamSynchronize(ctx->stream_hash);
    for (DevBuf &b : ctx->ws) if (b.p) cudaFree(b.p);
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    cudaEventDestroy(ctx->ev_a); cudaEventDestroy(ctx->ev_b); cudaEventDestroy(ctx->ev_fork); cudaEventDestroy(ctx->ev_join);
    cudaEventDestroy(ctx->ev_join2); cudaEventDestroy(ctx->ev_call0); cudaEventDestroy(ctx->ev_call1);
    for (int i = 0; i < 8; i++) { cudaEventDestroy(ctx->ev_grp[i]); cudaEventDestroy(ctx->ev_hram[i]); cudaEventDestroy(ctx->ev_prep[i][0]); cudaEventDestroy(ctx->ev_prep[i][1]); }
    cudaStreamDestroy(ctx->stream_hash);
    cudaStreamDestroy(ctx->stream); cudaStreamDestroy(ctx->stream2); cudaStreamDestroy(ctx->stream_copy); cudaStreamDestroy(ctx->stream3);
    delete ctx;
}

const char *dalek_b200_last_error(const dalek_b200_ctx *ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

int dalek_b200_set_option(dalek_b200_ctx *ctx, const char *name, long value)
{
    if (!ctx || !name) return DALEK_E_INVALID_ARG;
    if (!strcmp(name, "window_bits")) { if (value != 0 && (value < 4 || value > 20)) return DALEK_E_INVALID_ARG; ctx->opt_window_bits = value; return 0; }
    if (!strcmp(name, "host_chunks")) { if (value < 1 || value > 8) return DALEK_E_INVALID_ARG; ctx->opt_host_chunks = value; return 0; }
    if (!strcmp(name, "decompress_f64")) { ctx->opt_decompress_f64 = value ? 1 : 0; return 0; }
    if (!strcmp(name, "trace")) { ctx->opt_trace = value ? 1 : 0; return 0; }
    if (!strcmp(name, "precomp_tables")) { ctx->opt_precomp_tables = value ? 1 : 0; return 0; }
    if (!strcmp(name, "double_base_comb")) { ctx->opt_double_base_comb = value ? 1 : 0; return 0; }
    if (!strcmp(name, "dedupe_keys")) { ctx->opt_dedupe_keys = value ? 1 : 0; return 0; }
    if (!strcmp(name, "verify_pieces")) { if (value < 1 || value > 8) return DALEK_E_INVALID_ARG; ctx->opt_verify_pieces = value; return 0; }
    if (!strcmp(name, "transcript_warp")) { ctx->opt_transcript_warp = value ? 1 : 0; return 0; }
    if (!strcmp(name, "transcript_blocks")) { ctx->opt_transcript_blocks = value ? 1 : 0; return 0; }
    if (!strcmp(name, "bpt_group")) { ctx->opt_bpt_group = value ? 1 : 0; return 0; }
    if (!strcmp(name, "each_comb")) { if (value < 0 || value > 2) return DALEK_E_INVALID_ARG; ctx->opt_each_comb = value; return 0; }
    if (!strcmp(name, "small_straus")) { ctx->opt_small_straus = value ? 1 : 0; return 0; }
    if (!strcmp(name, "acc_tma")) { ctx->opt_acc_tma = value ? 1 : 0; return 0; }
    if (!strcmp(name, "field_f64")) { ctx->opt_field_f64 = value ? 1 : 0; return 0; }
    if (!strcmp(name, "verify_chunk")) { if (value < 0 || value > (1 << 20)) return DALEK_E_INVALID_ARG; ctx->opt_verify_chunk = value; return 0; }
    return DALEK_E_INVALID_ARG;
}

int dalek_b200_get_option(const dalek_b200_ctx *ctx, const char *name, long *value)
{
    if (!ctx || !name || !value) return DALEK_E_INVALID_ARG;
    const struct { const char *name; long v; } opts[] = {
        {"window_bits", ctx->opt_window_bits}, {"host_chunks", ctx->opt_host_chunks}, {"decompress_f64", ctx->opt_decompress_f64},
        {"trace", ctx->opt_trace}, {"precomp_tables", ctx->opt_precomp_tables}, {"double_base_comb", ctx->opt_double_base_comb},
        {"dedupe_keys", ctx->opt_dedupe_keys}, {"verify_pieces", ctx->opt_verify_pieces}, {"transcript_warp", ctx->opt_transcript_warp},
        {"transcript_blocks", ctx->opt_transcript_blocks}, {"each_comb", ctx->opt_each_comb}, {"bpt_group", ctx->opt_bpt_group}, {"small_straus", ctx->opt_small_straus},
        {"acc_tma", ctx->opt_acc_tma}, {"field_f64", ctx->opt_field_f64}, {"verify_chunk", ctx->opt_verify_chunk}};
    for (const auto &o : opts)
        if (!strcmp(name, o.name)) { *value = o.v; return 0; }
    return DALEK_E_INVALID_ARG;
}

uint64_t dalek_b200_launch_count(const dalek_b200_ctx *ctx) { return ctx ? ctx->launches : 0; }

int dalek_b200_last_kernel_ms(const dalek_b200_ctx *ctx, float *ms, int *launches)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    if (ms) *ms = ctx->last_kernel_ms;
    if (launches) *launches = ctx->last_kernel_launches;
    return 0;
}

int dalek_b200_last_stage_ms(const dalek_b200_ctx *ctx, const char *stage, float *ms)
{
    if (!ctx || !stage || !ms) return DALEK_E_INVALID_ARG;
    if (!strcmp(stage, "bucket_accumulate")) { *ms = ctx->last_kernel_ms; return 0; }
    if (!strcmp(stage, "decompress_R")) { *ms = ctx->last_prep_ms; return 0; }
    return DALEK_E_INVALID_ARG;
}

int dalek_b200_last_call_ms(const dalek_b200_ctx *ctx, float *ms)
{
    if (!ctx || !ms) return DALEK_E_INVALID_ARG;
    *ms = ctx->last_call_ms;
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
int msm_driver_ws_reserve(dalek_b200_ctx *ctx)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_WINDOWS], MSM_WINDOWS_MAX * sizeof(ge_p3_raw)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_MSM_RESULT], 3 * sizeof(MsmResult) + 64))) return rc;
    return ws_reserve(ctx, ctx->ws[WS_FLAGS], FLAG_WORDS * sizeof(int));
}

// Inputs (host or device) -> bucket sums -> window accumulators (-> result if d_result); the FLAG_STATUS word is set if
// a point does not decode.
// Host inputs are streamed in chunks on a dedicated copy stream: while chunk k+1 crosses PCIe,
// chunk k is converted, sorted and added into the (persistent) bucket sums.
static int run_msm(dalek_b200_ctx *ctx, const void *scalars, const void *points_in, bool on_device, int point_fmt, size_t n,
                   size_t n_window /* the size the window width is chosen from: n, or the shard size of a sharded MSM */,
                   ge_p3_raw *d_windows, MsmResult *d_result)
{
    int rc;
    const size_t pin = msm_point_bytes(point_fmt);
    cudaStream_t st = ctx->stream;
    const int c = msm_choose_window_bits(ctx, n_window);
    // the reference's dispatch (edwards.rs:1025-1029): below 190 points vartime Straus -- here three launches
    // (straus_vt.cu) instead of the ~27 of the bucket pipeline; only for whole MSMs (a shard must yield window sums)
    const bool straus = d_result && n == n_window && n < STRAUS_VT_THRESHOLD && ctx->opt_small_straus && ctx->opt_field_f64;
    // the bucket kernel reads affine Niels; Straus builds its own tables and keeps extended inputs projective, as an
    // inversion would only lengthen its latency-bound path
    const int kind = msm_prepared_kind(point_fmt, straus ? PK_PNIELS : PK_NIELS);
    const size_t psz = kind == PK_NIELS ? sizeof(ge_niels_packed) : sizeof(ge_pniels_packed);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], std::max<size_t>(1, n) * psz))) return rc;
    int *d_bad = (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_FLAGS].p, 0, FLAG_WORDS * sizeof(int), st));
    if (on_device) {
        if (straus) {
            if ((rc = msm_prepare_points(ctx, points_in, point_fmt, n, ctx->ws[WS_STAGING_OUT].p, d_bad, kind))) return rc;
            if ((rc = straus_vartime_msm(ctx, (const uint32_t *)scalars, ctx->ws[WS_STAGING_OUT].p, kind, n, d_result))) return rc;
        } else {
            // the point conversion (or decompression) runs on the second stream under the digit / sort passes of the main one
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
            CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
            if ((rc = msm_prepare_points_on(ctx, ctx->stream2, points_in, point_fmt, n, ctx->ws[WS_STAGING_OUT].p, d_bad))) return rc;
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
            if ((rc = msm_accumulate_chunk(ctx, (const uint32_t *)scalars, (const ge_niels_packed *)ctx->ws[WS_STAGING_OUT].p, n, c, true, 0, 0, ctx->ev_join))) return rc;
        }
    } else {
        if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n) * 32))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * pin))) return rc;
        int K = n >= (1u << 18) ? (int)std::min<long>(8, std::max<long>(1, ctx->opt_host_chunks)) : 1;
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream_copy, ctx->ev_fork, 0));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
        // equal pieces: every piece re-runs the per-bucket passes (scans, task lists) and revisits all bucket sums,
        // in exchange for more copy / compute overlap (tools/sweep_msm_options.py times 1, 2, 4 and 8 chunks)
        for (int k = 0; k < K; k++) {
            const size_t i0 = n * k / K, i1 = n * (k + 1) / K, cnt = i1 - i0;
            char *ds = (char *)ctx->ws[WS_SCALARS].p + i0 * 32, *dp = (char *)ctx->ws[WS_STAGING_IN].p + i0 * pin;
            if (cnt) {
                CUDA_TRY(ctx, cudaMemcpyAsync(ds, (const char *)scalars + i0 * 32, cnt * 32, cudaMemcpyHostToDevice, ctx->stream_copy));
                CUDA_TRY(ctx, cudaMemcpyAsync(dp, (const char *)points_in + i0 * pin, cnt * pin, cudaMemcpyHostToDevice, ctx->stream_copy));
            }
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_grp[k], ctx->stream_copy));
            CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_grp[k], 0));
            char *dq = (char *)ctx->ws[WS_STAGING_OUT].p + i0 * psz;
            if (straus) {                                            // K = 1 for small inputs
                if ((rc = msm_prepare_points(ctx, dp, point_fmt, cnt, dq, d_bad, kind))) return rc;
                if ((rc = straus_vartime_msm(ctx, (const uint32_t *)ds, dq, kind, cnt, d_result))) return rc;
            } else {
                // as for device inputs: the chunk's points are converted on the second stream while its digit / sort
                // passes run on the main one (the normalisation's inversions would otherwise sit on the critical path)
                CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_grp[k], 0));
                if ((rc = msm_prepare_points_on(ctx, ctx->stream2, dp, point_fmt, cnt, dq, d_bad))) return rc;
                CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
                if ((rc = msm_accumulate_chunk(ctx, (const uint32_t *)ds, (const ge_niels_packed *)dq, cnt, c, k == 0, 0, 0, ctx->ev_join))) return rc;
            }
        }
    }
    if (!straus && (rc = msm_reduce_finish(ctx, c, d_windows, d_result))) return rc;
    return 0;
}

int msm_read_result(dalek_b200_ctx *ctx, const MsmResult *d_result, const int *d_bad, const uint32_t *d_enc,
                    uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    int rc;
    cudaStream_t st = ctx->stream;
    if ((rc = pinned_reserve(ctx, sizeof(MsmResult) + 128))) return rc;
    MsmResult *h = (MsmResult *)ctx->h_pinned;
    int *h_bad = (int *)((char *)ctx->h_pinned + sizeof(MsmResult));
    uint8_t *h_enc = (uint8_t *)ctx->h_pinned + sizeof(MsmResult) + 64;
    CUDA_TRY(ctx, cudaMemcpyAsync(h, d_result, sizeof(MsmResult), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(h_bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (d_enc) CUDA_TRY(ctx, cudaMemcpyAsync(h_enc, d_enc, 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    if (out_compressed) memcpy(out_compressed, d_enc ? h_enc : (const uint8_t *)h->compressed, 32);
    if (out_limbs) memcpy(out_limbs, h->limbs, 160);
    return *h_bad ? DALEK_NONE : DALEK_OK;
}

// One whole MSM on the context's device, read back.  Ristretto points also give the Ristretto encoding of the result in
// out_compressed.
int msm_whole(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt, size_t n,
              uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    int rc;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    MsmResult *d_res = (MsmResult *)ctx->ws[WS_MSM_RESULT].p;
    uint32_t *d_enc = point_fmt == DALEK_POINTS_RISTRETTO ? (uint32_t *)(d_res + 1) : nullptr;
    if ((rc = run_msm(ctx, scalars, points, on_device, point_fmt, n, n, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, d_res))) return rc;
    if (d_enc && (rc = ristretto_encode_result(ctx, d_res, d_enc))) return rc;
    return msm_read_result(ctx, d_res, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS, d_enc, out_compressed, out_limbs);
}

// The public entry points check the point format.
static int msm_common(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt,
                      size_t n, uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!ctx || (n && (!scalars || !points)) || n >= (1ull << 31)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    return msm_whole(ctx, scalars, points, on_device, point_fmt, n, out_compressed, out_limbs);
}

static bool edwards_format(int point_fmt) { return point_fmt == DALEK_POINTS_COMPRESSED || point_fmt == DALEK_POINTS_EXTENDED; }

extern "C" {

int dalek_b200_edwards_vartime_msm(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points, int point_fmt,
                                   size_t n, uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!edwards_format(point_fmt)) return DALEK_E_INVALID_ARG;
    return msm_common(ctx, scalars, points, false, point_fmt, n, out_compressed, out_limbs);
}

int dalek_b200_edwards_vartime_msm_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points, int point_fmt,
                                       size_t n, uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!edwards_format(point_fmt)) return DALEK_E_INVALID_ARG;
    return msm_common(ctx, d_scalars, d_points, true, point_fmt, n, out_compressed, out_limbs);
}

int dalek_b200_ristretto_vartime_msm(dalek_b200_ctx *ctx, const uint8_t *scalars, const uint8_t *points, size_t n,
                                     uint8_t out_compressed[32])
{
    if (!out_compressed) return DALEK_E_INVALID_ARG;
    return msm_common(ctx, scalars, points, false, DALEK_POINTS_RISTRETTO, n, out_compressed, nullptr);
}

int dalek_b200_msm_window_count(dalek_b200_ctx *ctx, size_t n_shard)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    return msm_window_count_for_bits(msm_choose_window_bits(ctx, n_shard));
}

size_t dalek_b200_msm_partial_bytes(dalek_b200_ctx *ctx, size_t n_shard)
{
    if (!ctx) return 0;
    return (size_t)msm_window_count_for_bits(msm_choose_window_bits(ctx, n_shard)) * 160 + 8;
}

void *dalek_b200_stream(dalek_b200_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

}  // extern "C"

// A shard's record as it crosses the boundary (and the exchange between ranks): the window accumulators as
// canonical radix-2^51 limbs (20 u64 each, window 0 = least significant) followed by one u64 status word
// (non-zero: a compressed point of the shard did not decode).
__global__ void k_windows_to_record(const ge_p3_raw *__restrict__ win, int nwin, const int *__restrict__ bad, uint64_t *__restrict__ out)
{
    int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w == nwin) out[20 * (size_t)nwin] = (uint64_t)(*bad != 0);
    if (w >= nwin) return;
    ge_p3 p; ge_p3_raw r = win[w]; ge_p3_load_raw(p, r);
    fe_to_limbs51(out + 20 * w, p.X); fe_to_limbs51(out + 20 * w + 5, p.Y);
    fe_to_limbs51(out + 20 * w + 10, p.Z); fe_to_limbs51(out + 20 * w + 15, p.T);
}
// `ranks` records of `rec_words` u64 each -> ranks x nwin raw accumulators; *any_bad |= status words
__global__ void k_records_to_windows(const uint64_t *__restrict__ in, int ranks, int nwin, size_t rec_words,
                                     ge_p3_raw *__restrict__ win, int *__restrict__ any_bad)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ranks * nwin) return;
    const int r = t / nwin, w = t % nwin;
    const uint64_t *src = in + (size_t)r * rec_words + 20 * (size_t)w;
    ge_p3 p;
    fe_from_limbs51(p.X, src); fe_from_limbs51(p.Y, src + 5); fe_from_limbs51(p.Z, src + 10); fe_from_limbs51(p.T, src + 15);
    ge_p3_raw o; ge_p3_store_raw(o, p); win[t] = o;
    if (w == 0 && rec_words > 20 * (size_t)nwin && in[(size_t)r * rec_words + 20 * (size_t)nwin]) atomicOr(any_bad, 1);
}

// Enqueue the partial MSM of one shard on the context's stream and leave its record (window accumulators +
// status word) in WS_SHARD_RECORD, where ..._partial_async copies it out; nothing is synchronised.  ev_a .. ev_b bracket the bucket accumulation.
static int partial_enqueue(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt,
                           size_t n_local, size_t n_shard, int *nwin_out)
{
    if (!ctx || (n_local && (!scalars || !points)) || n_local > n_shard || !edwards_format(point_fmt) || n_local >= (1ull << 31))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    const int c = msm_choose_window_bits(ctx, n_shard);
    const int nwin = msm_window_count_for_bits(c);
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SHARD_RECORD], (size_t)nwin * 160 + 8))) return rc;
    if ((rc = run_msm(ctx, scalars, points, on_device, point_fmt, n_local, n_shard, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, nullptr))) return rc;
    k_windows_to_record<<<(nwin + 1 + 63) / 64, 64, 0, ctx->stream>>>((const ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, nwin, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS,
                                                                     (uint64_t *)ctx->ws[WS_SHARD_RECORD].p);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    *nwin_out = nwin;
    return 0;
}

static void read_kernel_ms(dalek_b200_ctx *ctx)
{
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
}

static int partial_common(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt,
                          size_t n_local, size_t n_shard, uint64_t *out_windows)
{
    if (!ctx || !out_windows) return DALEK_E_INVALID_ARG;
    CallTimer timer(ctx);
    int rc, nwin = 0;
    if ((rc = partial_enqueue(ctx, scalars, points, on_device, point_fmt, n_local, n_shard, &nwin))) return rc;
    const size_t bytes = (size_t)nwin * 160 + 8;
    if ((rc = pinned_reserve(ctx, bytes))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws[WS_SHARD_RECORD].p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    read_kernel_ms(ctx);
    memcpy(out_windows, ctx->h_pinned, (size_t)nwin * 160);
    uint64_t status; memcpy(&status, (const char *)ctx->h_pinned + (size_t)nwin * 160, 8);
    return status ? DALEK_NONE : DALEK_OK;
}

// dst_device >= 0: d_out_record lives on that (other) device -- the record crosses NVLink as a peer copy
int msm_partial_enqueue_record(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt,
                               size_t n_local, size_t n_shard, void *d_out_record, int dst_device)
{
    if (!ctx || !d_out_record) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_call0, ctx->stream));     // the device span ends in ..._combine_dev
    ctx->async_open = true;
    int rc, nwin = 0;
    if ((rc = partial_enqueue(ctx, scalars, points, on_device, point_fmt, n_local, n_shard, &nwin))) return rc;
    if (dst_device >= 0 && dst_device != ctx->device)
        CUDA_TRY(ctx, cudaMemcpyPeerAsync(d_out_record, dst_device, ctx->ws[WS_SHARD_RECORD].p, ctx->device, (size_t)nwin * 160 + 8, ctx->stream));
    else
        CUDA_TRY(ctx, cudaMemcpyAsync(d_out_record, ctx->ws[WS_SHARD_RECORD].p, (size_t)nwin * 160 + 8, cudaMemcpyDeviceToDevice, ctx->stream));
    return DALEK_OK;
}

// records (host or device) -> Horner over windows -> result read-back.  Not msm_read_result: the device span of an
// open ..._partial_async call ends after the read-back copies, and only such a call refreshes last_kernel_ms.
int msm_combine_records(dalek_b200_ctx *ctx, const void *records, bool on_device, size_t rec_bytes, int ranks, size_t n_shard,
                        uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!ctx || !records || ranks < 1 || ranks > 1024) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    const int c = msm_choose_window_bits(ctx, n_shard);
    const int nwin = msm_window_count_for_bits(c);
    const size_t cnt = (size_t)ranks * nwin;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_COMBINE_WINDOWS], cnt * sizeof(ge_p3_raw)))) return rc;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    if ((rc = pinned_reserve(ctx, sizeof(MsmResult) + 64))) return rc;
    cudaStream_t st = ctx->stream;
    const void *d_rec = records;
    if (!on_device) {
        if ((rc = ws_reserve(ctx, ctx->ws[WS_COMBINE_RECORDS], (size_t)ranks * rec_bytes))) return rc;
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_COMBINE_RECORDS].p, records, (size_t)ranks * rec_bytes, cudaMemcpyHostToDevice, st));
        d_rec = ctx->ws[WS_COMBINE_RECORDS].p;
    }
    int *d_bad = (int *)ctx->ws[WS_FLAGS].p + FLAG_COMBINE;
    CUDA_TRY(ctx, cudaMemsetAsync(d_bad, 0, 4, st));
    k_records_to_windows<<<(unsigned)((cnt + 63) / 64), 64, 0, st>>>((const uint64_t *)d_rec, ranks, nwin, rec_bytes / 8,
                                                                      (ge_p3_raw *)ctx->ws[WS_COMBINE_WINDOWS].p, d_bad);
    ctx->launches++;
    if ((rc = msm_combine_windows(ctx, (const ge_p3_raw *)ctx->ws[WS_COMBINE_WINDOWS].p, ranks, nwin, c, (MsmResult *)ctx->ws[WS_MSM_RESULT].p))) return rc;
    MsmResult *h = (MsmResult *)ctx->h_pinned;
    int *h_bad = (int *)((char *)ctx->h_pinned + sizeof(MsmResult));
    CUDA_TRY(ctx, cudaMemcpyAsync(h, ctx->ws[WS_MSM_RESULT].p, sizeof(MsmResult), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(h_bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
    if (ctx->async_open) CUDA_TRY(ctx, cudaEventRecord(ctx->ev_call1, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    if (ctx->async_open) {
        float ms = 0.f;
        if ((ms = elapsed_ms(ctx->ev_call0, ctx->ev_call1)) >= 0.f) ctx->last_call_ms = ms;
        read_kernel_ms(ctx);                                     // the bucket kernels of the partial call
        ctx->async_open = false;
    }
    if (out_compressed) memcpy(out_compressed, h->compressed, 32);
    if (out_limbs) memcpy(out_limbs, h->limbs, 160);
    return *h_bad ? DALEK_NONE : DALEK_OK;
}

extern "C" {

int dalek_b200_edwards_msm_partial(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points, int point_fmt,
                                   size_t n_local, size_t n_shard, uint64_t *out_windows)
{
    return partial_common(ctx, scalars, points, false, point_fmt, n_local, n_shard, out_windows);
}

int dalek_b200_edwards_msm_partial_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points, int point_fmt,
                                       size_t n_local, size_t n_shard, uint64_t *out_windows)
{
    return partial_common(ctx, d_scalars, d_points, true, point_fmt, n_local, n_shard, out_windows);
}

int dalek_b200_edwards_msm_partial_async(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points, int point_fmt,
                                         size_t n_local, size_t n_shard, void *d_out_record)
{
    return msm_partial_enqueue_record(ctx, scalars, points, false, point_fmt, n_local, n_shard, d_out_record, -1);
}

int dalek_b200_edwards_msm_partial_dev_async(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points, int point_fmt,
                                             size_t n_local, size_t n_shard, void *d_out_record)
{
    return msm_partial_enqueue_record(ctx, d_scalars, d_points, true, point_fmt, n_local, n_shard, d_out_record, -1);
}

int dalek_b200_edwards_msm_combine(dalek_b200_ctx *ctx, const uint64_t *windows, int ranks, size_t n_shard,
                                   uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    const size_t rec = (size_t)msm_window_count_for_bits(msm_choose_window_bits(ctx, n_shard)) * 160;   // no status words
    return msm_combine_records(ctx, windows, false, rec, ranks, n_shard, out_compressed, out_limbs);
}

int dalek_b200_edwards_msm_combine_dev(dalek_b200_ctx *ctx, const void *d_records, int ranks, size_t n_shard,
                                       uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    return msm_combine_records(ctx, d_records, true, dalek_b200_msm_partial_bytes(ctx, n_shard), ranks, n_shard, out_compressed, out_limbs);
}

}  // extern "C"
