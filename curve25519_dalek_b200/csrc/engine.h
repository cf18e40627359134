// engine.h -- internal (C++) interface between the translation units of libdalek_b200.so.
// The public boundary is include/dalek_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "../../include/dalek_b200.h"
#include "ge.cuh"

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

struct dalek_b200_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;
    cudaStream_t stream_copy = nullptr;
    cudaStream_t stream3 = nullptr;      // second transcript chain (odd verify pieces)
    cudaStream_t stream_hash = nullptr;  // SHA-512 of every verify piece: never queued behind a transcript (a long dependent chain)
    cudaEvent_t ev_hram[8] = {};         // "hram of piece k done" (stream_hash)
    cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_fork = nullptr, ev_join = nullptr, ev_join2 = nullptr;
    cudaEvent_t ev_call0 = nullptr, ev_call1 = nullptr;   // device span of the last hot-path call (CallTimer)
    cudaEvent_t ev_prep[8][2] = {};      // around the R-decompression kernel of each verify_batch piece (stream2)
    int prep_pieces = 0;
    float last_prep_ms = 0.f;            // their sum in the last verify_batch call
    cudaEvent_t ev_grp[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // one per input piece
    std::string last_error;
    uint64_t launches = 0;
    // options
    long opt_window_bits = 0;
    long opt_verify_chunk = 0;     // 0: the reference's single transcript over the whole batch; k > 0: opt-in, one transcript per k signatures
    long opt_host_chunks = 8;   // host-buffer MSM calls stream the pairs in this many chunks (copy/compute overlap)
    long opt_trace = 0;            // 1: print a per-stage device timeline of verify_batch calls to stderr (diagnostics)
    long opt_precomp_tables = 0;   // 1: precomputations of >= 4096 points also keep 2^(cw) P tables (one bucket window, no doublings)
    long opt_double_base_comb = 1; // double-base batch through the shared-memory fixed-base comb (0 = per-pair Straus)
    long opt_dedupe_keys = 1;   // verify_batch decompresses every distinct public key once
    long opt_verify_pieces = 4; // host-buffer verify_batch calls stream the signatures in this many pieces
    long opt_decompress_f64 = 1; // square-root exponentiation of point decompression on the FP64-pipe field
    long opt_acc_tma = 0;       // bucket kernel gathers points with TMA bulk copies + mbarriers instead of cp.async (A/B option)
    long opt_transcript_warp = 1; // up to 2048 Merlin transcripts per launch run one WARP each (25-lane Keccak); 0 = one thread each
    long opt_transcript_blocks = 1; // more transcripts than that: one THREAD each with the rate block staged in shared memory (0 = byte-wise sponge)
    long opt_each_comb = 1;     // verify_each: 1 = per-key comb tables when every key signs >= 8 signatures on average, 2 = always, 0 = never
    long opt_small_straus = 1;  // fewer than 190 pairs: vartime Straus (3 launches) instead of the bucket pipeline
    long opt_field_f64 = 1;     // bucket kernel on the FP64 pipe (fe64.cuh) instead of IMAD.WIDE (fe.cuh)
    // timing of the dominant kernel in the last call
    float last_kernel_ms = 0.f;
    float last_call_ms = 0.f;
    int last_kernel_launches = 0;
    bool async_open = false;       // a ..._partial_async call is in flight: its device span ends in ..._combine_dev
    // device workspaces (grown on demand, reused across calls)
    DevBuf scalars, points_in, points, digits, counts, offsets, sorted, buckets, red_a, red_b, red_c,
        red_d, key_pts, result, flags, misc0, misc1, misc2, misc3, misc4, misc5, zs, base_table, ntasks, task_off, tasks, task_sums, msg_offs, sum_desc, sum_part, key_table, key_acc, task_order, sig_status, misc6, each_pow, each_tab, each_kstat;
    DevBuf prep_prod;   // extended-point preparation: the Z product of each group of points (then its inverse), and running products
    uint32_t hash_seed[4] = {0x243F6A88u, 0x85A308D3u, 0x13198A2Eu, 0x03707344u};   // key of the public-key de-duplication hash, redrawn per context
    int sum_desc_c = -1;
    bool base_table_ready = false;
    bool each_attr_set = false;     // the same for k_verify_each_comb
    bool comb_attr_set = false;     // cudaFuncAttributeMaxDynamicSharedMemorySize set for the comb kernel on this device
    bool sort_attr_set = false;     // the same for the two digit-sort kernels of msm.cu, at their call-independent bounds
    DevBuf comb_base_table;         // comb table of the Ed25519 basepoint (comb.cuh) for X25519 public keys and signing, built once
    bool comb_base_table_ready = false;
    DevBuf mb_ws[2];                // batched MSMs (msm_batch.cu): the workspace of the pieces on each of the two streams
    // pinned host staging
    void *h_pinned = nullptr;
    size_t h_pinned_cap = 0;
    size_t last_zs_n = 0;
    std::vector<std::pair<const char *, cudaEvent_t>> trace;   // stage marks of the current call (opt_trace)
};

#define CUDA_TRY(ctx, expr)                                                                      \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            (ctx)->last_error = std::string(#expr) + ": " + cudaGetErrorString(_e);              \
            return -3;                                                                           \
        }                                                                                        \
    } while (0)

// Milliseconds between two events, or a negative value if either was never recorded / has not completed; a failure does
// not stay behind as the context's "last CUDA error" (a later cudaGetLastError() would report it for an innocent call).
inline float elapsed_ms(cudaEvent_t a, cudaEvent_t b)
{
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, a, b) == cudaSuccess) return ms;
    cudaGetLastError();
    return -1.f;
}

// Device time of one blocking call: an event on the main stream at entry, one after everything the call enqueued
// (the other streams are joined into the main one before a call returns); read with dalek_b200_last_call_ms.
struct CallTimer {
    dalek_b200_ctx *ctx;
    explicit CallTimer(dalek_b200_ctx *c) : ctx(c) { if (ctx) cudaEventRecord(ctx->ev_call0, ctx->stream); }
    ~CallTimer()
    {
        if (!ctx) return;
        float ms = 0.f;
        if (cudaEventRecord(ctx->ev_call1, ctx->stream) == cudaSuccess && cudaEventSynchronize(ctx->ev_call1) == cudaSuccess &&
            (ms = elapsed_ms(ctx->ev_call0, ctx->ev_call1)) >= 0.f)
            ctx->last_call_ms = ms;
    }
};

// diagnostics: timestamp `name` on `st` (relative to the CallTimer start), printed by trace_dump
inline void trace_mark(dalek_b200_ctx *ctx, const char *name, cudaStream_t st)
{
    if (!ctx->opt_trace) return;
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    cudaEventRecord(e, st);
    ctx->trace.push_back({name, e});
}
inline void trace_dump(dalek_b200_ctx *ctx)
{
    if (!ctx->opt_trace) return;
    cudaDeviceSynchronize();
    for (auto &m : ctx->trace) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ctx->ev_call0, m.second);
        fprintf(stderr, "[trace] %8.3f ms  %s\n", ms, m.first);
        cudaEventDestroy(m.second);
    }
    ctx->trace.clear();
}

// The rule for flat messages of the host-buffer calls (include/dalek_b200.h, hash to group): for n > 0 the n + 1 offsets
// start at 0 and do not decrease, and msgs_flat may be NULL only when every message is empty.  A negative length would
// read outside the staging buffer.
inline bool flat_messages_ok(const uint8_t *msgs_flat, const uint64_t *offsets, size_t n)
{
    if (!n) return true;
    if (!offsets || offsets[0] != 0) return false;
    for (size_t i = 0; i < n; i++)
        if (offsets[i] > offsets[i + 1]) return false;
    return msgs_flat || offsets[n] == 0;
}

int ws_reserve(dalek_b200_ctx *ctx, DevBuf &b, size_t bytes);
int pinned_reserve(dalek_b200_ctx *ctx, size_t bytes);

// ---- point preparation (msm.cu) ----
// kinds of prepared device point arrays: the bucket kernel reads PK_NIELS only; the vartime Straus path takes either
enum { PK_NIELS = 0 /* ge_niels_packed, 96 B */, PK_PNIELS = 1 /* ge_pniels_packed, 128 B */ };

// Bytes per input point of a format DALEK_POINTS_*: 32 for the compressed Edwards and Ristretto encodings, 160 for
// extended limbs.
inline size_t msm_point_bytes(int point_fmt) { return point_fmt == DALEK_POINTS_EXTENDED ? 160 : 32; }

// Convert n input points (device memory, format DALEK_POINTS_*) into packed Niels form.
// Compressed Edwards and Ristretto inputs give affine Niels (decoding yields Z = 1) and set *d_bad (device int) nonzero
// if any fails to decode.  Extended inputs give affine Niels too, normalised to Z = 1 with one inversion per call (three
// launches on the given stream, with the context's prep_prod workspace);
// with kind = PK_PNIELS they give projective Niels instead (no inversion, for the latency-bound Straus path).
// msm_prepared_kind tells which kind a format and a requested kind give.
int msm_prepare_points(dalek_b200_ctx *ctx, const void *d_in, int point_fmt, size_t n, void *d_out,
                       int *d_bad, int kind = PK_NIELS);
int msm_prepared_kind(int point_fmt, int kind);

// Window width (bits) the engine uses for an MSM over n pairs.
int msm_choose_window_bits(const dalek_b200_ctx *ctx, size_t n);
int msm_window_count_for_bits(int c);

// total = sum over ranks of windows, Horner-combined; writes compressed (8 words) + canonical
// limbs51 (20 u64) + identity flag to d_result (layout: 8 u32 | pad | 20 u64 | u32 flag).
struct MsmResult { uint32_t compressed[8]; uint64_t limbs[20]; uint32_t is_identity; uint32_t pad; };
// building blocks: one chunk of pairs into the buckets; then reduction (+ Horner + encode if d_result)
// points_ready (optional): an event after which d_points may be read -- the digit and sort passes do not wait for it
int msm_accumulate_chunk(dalek_b200_ctx *ctx, const uint32_t *d_scalars, const ge_niels_packed *d_points, size_t n,
                         int c, bool first, int active_windows = 0, size_t flat = 0, cudaEvent_t points_ready = nullptr);
int msm_prepare_points_on(dalek_b200_ctx *ctx, cudaStream_t st, const void *d_in, int point_fmt, size_t n, void *d_out, int *d_bad,
                          int kind = PK_NIELS);
// window width for `n_short` scalars of `short_bits` bits plus `n_long` full-width scalars (verify_batch)
int msm_choose_window_bits_mixed(const dalek_b200_ctx *ctx, size_t n_short, int short_bits, size_t n_long);
int msm_reduce_finish(dalek_b200_ctx *ctx, int c, ge_p3_raw *d_windows, MsmResult *d_result, bool flat = false);
int msm_combine_windows(dalek_b200_ctx *ctx, const ge_p3_raw *d_windows, int ranks, int nwin, int c,
                        MsmResult *d_result);
// Blocking read-back of an MSM enqueued on ctx->stream (api.cu): the MsmResult at d_result, the status flag at d_bad
// and, if d_enc is given, the 32-byte Ristretto encoding at d_enc, which then goes to out_compressed instead of the
// Edwards one.  Sets last_kernel_ms from ev_a .. ev_b and fills the non-null outputs.  Returns DALEK_NONE if the flag
// is set (a point did not decode), else DALEK_OK, or a negative engine code.
int msm_read_result(dalek_b200_ctx *ctx, const MsmResult *d_result, const int *d_bad, const uint32_t *d_enc,
                    uint8_t out_compressed[32], uint64_t out_limbs[20]);

// One whole vartime MSM (api.cu), host or device inputs, enqueued on ctx->stream and read back: what the single-MSM entry
// points run after their argument checks.  Returns DALEK_OK, DALEK_NONE or a negative engine code.
int msm_whole(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt, size_t n,
              uint8_t out_compressed[32], uint64_t out_limbs[20]);

// ---- sharded MSM building blocks (api.cu), shared with the single-process multi-GPU entry points (multi.cu) ----
// Enqueue the MSM of one shard on ctx's stream; its record (window accumulators + status word) is copied to
// d_out_record (on device dst_device if >= 0 and different from ctx's: a peer copy).  Nothing is synchronised.
int msm_partial_enqueue_record(dalek_b200_ctx *ctx, const void *scalars, const void *points, bool on_device, int point_fmt,
                               size_t n_local, size_t n_shard, void *d_out_record, int dst_device);
// `ranks` records (host or device, rec_bytes apart) -> per-window sums, Horner, encode; blocks for the result.
int msm_combine_records(dalek_b200_ctx *ctx, const void *records, bool on_device, size_t rec_bytes, int ranks, size_t n_shard,
                        uint8_t out_compressed[32], uint64_t out_limbs[20]);

// ---- front end of verify_batch reused by the per-signature verifier (batch.cu -> single.cu) ----
struct EachFront { const uint32_t *hs; const uint8_t *bad_s; const uint32_t *rep, *dense, *uniq; size_t nkeys; };
struct Sha512Prefix;   // hash.cuh: the dom2 prefix of Ed25519ph
int verify_each_front(dalek_b200_ctx *ctx, const uint8_t *d_msgs, const uint64_t *d_offs, const uint32_t *d_sigs, const uint32_t *d_keys,
                      size_t n, EachFront *out, const Sha512Prefix *ph_dom = nullptr);

// ---- variable-time Straus for small inputs (straus_vt.cu): the reference's path below 190 points ----
#define STRAUS_VT_THRESHOLD 190            // edwards.rs:1025-1029
int straus_vartime_msm(dalek_b200_ctx *ctx, const uint32_t *d_scalars, const void *d_points, int point_kind, size_t n,
                       MsmResult *d_result);

// ---- constant-time Straus (straus.cu) ----
int straus_ct_msm(dalek_b200_ctx *ctx, const uint32_t *d_scalars, const void *d_points_pniels, size_t n,
                  MsmResult *d_result);
// ---- fixed-base table (base.cu): 64 x 8 affine Niels entries (j+1) 16^i B, built once per context ----
int base_table_ensure(dalek_b200_ctx *ctx);
// ---- constant-time comb table of B (x25519.cu): 64 x 8 x COMB_ENTRY balanced FP64 doubles (comb.cuh), built once per
// context and shared by the X25519 public keys and the Ed25519 signer (sign.cu) ----
#define COMB_BASE_DOUBLES (64 * 8 * 15)
int comb_base_table_ensure(dalek_b200_ctx *ctx);

// RistrettoPoint::compress of an MSM result (straus.cu): 8 words at d_enc
int ristretto_encode_result(dalek_b200_ctx *ctx, const MsmResult *d_res, uint32_t *d_enc);
