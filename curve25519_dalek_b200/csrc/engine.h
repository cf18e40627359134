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

// The device workspaces of a context, one per role: the array ws indexed by WsRole.  Each comment names the files that
// may use the role, the owner first, then its lifetime in brackets: [call] the contents are valid within one public call,
// [cross-call] they survive until the named later call, [context] built once and kept.  Roles that only hold storage for
// one call are shared by the families listed; everything that must survive a call, is live while another role of the
// same files is, or is read by a nested call has a role of its own.  Workspaces grow on demand (ws_reserve) and are
// reused across calls; WS_FLAGS, WS_MSM_WINDOWS and WS_MSM_RESULT are reserved at their bounds by msm_driver_ws_reserve.
// tests/test_workspace_roles.py checks the file lists against the sources.
enum WsRole {
    // ---- per-item staging of one call, shared by every family that stages items ----
    // api.cu, base.cu, batch.cu, precomp.cu, scalars.cu, sign.cu, straus.cu [call] 32-byte scalars (MSM scalars, verify's
    // MSM coefficients, the signer's seeds, the results of the scalar batch calls)
    WS_SCALARS,
    // pieces.h, api.cu, base.cu, batch.cu, lizard.cu, point_ops.cu, precomp.cu, scalars.cu, sign.cu, single.cu, straus.cu,
    // varmul.cu [call] fixed-width inputs staged from the host: MSM input points, signatures and keys, the inputs of
    // run_pieces, the points of a segmented sum, the secret keys a signing-key set is built from
    WS_STAGING_IN,
    // pieces.h, api.cu, batch.cu, lizard.cu, point_ops.cu, precomp.cu, scalars.cu, straus.cu, varmul.cu [call] outputs of
    // run_pieces and the prepared Niels points of an MSM (verify's MSM points)
    WS_STAGING_OUT,
    // pieces.h, base.cu, batch.cu, scalars.cu, single.cu, straus.cu [call] flat messages (or fixed-stride prehashes) at
    // their own offsets; calls that stage no messages keep one-call per-item scratch here: compressed outputs (base.cu),
    // group products of the scalar inversion (scalars.cu), the decoded Niels points of the constant-time MSM (straus.cu)
    WS_STAGING_MSGS,
    // pieces.h, batch.cu, single.cu [call] the n + 1 message offsets of WS_STAGING_MSGS
    WS_MSG_OFFSETS,
    // double_base.cu, lizard.cu, montgomery.cu, point_ops.cu, scalars.cu, sign.cu, straus.cu, varmul.cu [call] small
    // per-call scratch: status words (the bad-index word of a signing-key set call), broadcast operands and tables, the
    // G/H tables of the Ristretto double-base batch
    WS_CALL_SCRATCH,
    // ---- tables built once per context ----
    // base.cu, double_base.cu, single.cu [context] 64 x 8 affine Niels entries (j+1) 16^i B (base_table_ensure)
    WS_BASE_TABLE,
    // x25519.cu, sign.cu [context] comb table of B in balanced FP64 doubles (comb_base_table_ensure)
    WS_COMB_BASE_TABLE,
    // ---- the MSM drivers ----
    // api.cu, batch.cu, precomp.cu, scalars.cu, straus.cu [call] status words; slots FLAG_*
    WS_FLAGS,
    // api.cu, batch.cu, precomp.cu [call] the window accumulators of one MSM (MSM_WINDOWS_MAX ge_p3_raw), read by
    // msm_reduce_finish
    WS_MSM_WINDOWS,
    // api.cu, batch.cu, precomp.cu, straus.cu [call] MSM results: up to three MsmResult and a 32-byte Ristretto encoding
    WS_MSM_RESULT,
    // api.cu [cross-call] a shard's record (nwin x 160 B + status word), from ..._partial_async until ..._combine_dev
    WS_SHARD_RECORD,
    // api.cu [call] the host records of msm_combine_records, staged
    WS_COMBINE_RECORDS,
    // api.cu [call] the ranks x nwin window accumulators of msm_combine_records
    WS_COMBINE_WINDOWS,
    // msm_batch.cu [call] the workspace of the pieces on the main stream
    WS_MSM_BATCH_0,
    // msm_batch.cu [call] the workspace of the pieces on the second stream
    WS_MSM_BATCH_1,
    // ---- group operations (point_ops.cu) ----
    // point_ops.cu [call] extended results before their shared-inversion encoding; the segmented sum's decoded points,
    // chunk plans, partial sums and results
    WS_POINT_OPS,
    // ---- scalar arithmetic (scalars.cu) ----
    // scalars.cu [call] the scalar Sum / Product: chunk plans, partial sums or products, results
    WS_SCALAR_FOLD,
    // ---- resident basepoint tables (varmul.cu) ----
    // varmul.cu [call] the items of a many-table multiplication grouped by table: a count per table for each of the two
    // streams, then the order of the items
    WS_BPT_ORDER,
    // ---- the MSM engine (msm.cu) and the Straus paths that stand in for it ----
    // msm.cu [call] extended-point preparation: the Z product of each group of points (then its inverse), running products
    WS_PREP_PROD,
    // msm.cu, straus_vt.cu [call] the digit sort's records, 8 B per non-zero digit; the NAF digits of the vartime Straus MSM
    WS_MSM_DIGITS,
    // msm.cu [call] the sorted point indices
    WS_MSM_SORTED,
    // msm.cu [call] bucket counts | coarse counts | heavy list
    WS_MSM_COUNTS,
    // msm.cu [call] bucket offsets | scan part sums | coarse bin cursors | extra-slice prefix and counts
    WS_MSM_OFFSETS,
    // msm.cu [call] tasks per bucket
    WS_MSM_NTASKS,
    // msm.cu [call] first task of each bucket | each window's base
    WS_MSM_TASK_OFF,
    // msm.cu [call] the tasks (bucket, first entry)
    WS_MSM_TASKS,
    // msm.cu [call] one partial sum per task
    WS_MSM_TASK_SUMS,
    // msm.cu [call] task length histogram | cursor | start | order
    WS_MSM_TASK_ORDER,
    // msm.cu, straus.cu [call] bucket sums (persistent over the chunks of one call); the per-point accumulators of the
    // constant-time Straus MSM
    WS_MSM_BUCKETS,
    // msm.cu, straus.cu, straus_vt.cu [call] the bucket reduction's pool of running sums; the Straus paths' tables or
    // partial sums
    WS_MSM_REDUCE_POOL,
    // msm.cu, straus_vt.cu [call] per-window sums of the reduction; the vartime Straus MSM's per-warp results
    WS_MSM_REDUCE_SUMS,
    // msm.cu [cross-call] the reduction's sum descriptors, kept while the width they were built for (sum_desc_c) repeats
    WS_MSM_SUM_DESC,
    // msm.cu [call] the first stage of the reduction's plain sums
    WS_MSM_SUM_PART,
    // ---- verification (batch.cu) and the per-signature verifier (single.cu) ----
    // batch.cu, sign.cu [call] SHA-512(R || A || M), 64 B per signature; in a sign call the signer's expanded keys (a
    // hazmat call: the caller's ExpandedSecretKey bytes)
    WS_VERIFY_HRAM,
    // batch.cu, sign.cu [call] h_i (z_i h_i once merged), 32 B per signature, read by single.cu after verify_each_front;
    // in a sign call the signer's verifying keys (a hazmat call: the caller's)
    WS_VERIFY_H,
    // batch.cu [call] z_i s_i
    WS_VERIFY_ZS_PROD,
    // batch.cu [cross-call] the 128-bit z_i, until the next verify call (ed25519_b200_last_zs)
    WS_VERIFY_Z,
    // batch.cu [call] partial sums of the z_i s_i
    WS_VERIFY_SUMS,
    // batch.cu [call] key de-duplication: hash table | rep | uniq | dense | counters, read by single.cu after
    // verify_each_front
    WS_VERIFY_KEY_TABLE,
    // batch.cu [call] per-key sums of z_i h_i over a range of signatures
    WS_VERIFY_KEY_ACC,
    // batch.cu [call] failure marks per signature (s, R) and per key, read by single.cu after verify_each_front
    WS_VERIFY_MARKS,
    // batch.cu [call] the callers' decompressed key points, staged
    WS_VERIFY_KEY_POINTS,
    // batch.cu [call] the small-order sum of each batch of a verify_batches call
    WS_BATCH_TORSION,
    // batch.cu, single.cu [call] one status byte per batch (verify_batches) or per signature (verify_each)
    WS_ITEM_STATUS,
    // single.cu [call] per-key comb tables of verify_each and of a verifying-key set's build: the 16^i A powers of each key
    WS_EACH_POW,
    // single.cu [call] per-key comb tables of verify_each: the tables
    WS_EACH_TABLES,
    // single.cu [call] per-key comb tables of verify_each: each key's status
    WS_EACH_KEY_STATUS,
    // single.cu [call] a verifying-key set call: the bad-index status word, then per signature h_i, the checked key index
    // and the non-canonical-s mark
    WS_KEY_SET_FRONT,
    WS_COUNT
};

// Slots (int words) of WS_FLAGS.  A call clears the slots it uses before its kernels write them.
enum {
    FLAG_STATUS = 0,    // an MSM input point did not decode; a zero scalar in a batch inversion (scalars.cu)
    FLAG_BAD_A = 0,     // verify: a public key did not decode
    FLAG_BAD_S = 1,     // verify: an s was not canonical
    FLAG_BAD_R = 2,     // verify: an R did not decode
    FLAG_COMBINE = 8,   // msm_combine_records: a record's status word; apart from FLAG_STATUS, which a partial call in
                        // flight still reads
    FLAG_WORDS = 16
};

// window accumulators of an MSM at the narrowest window width, c = 4 (msm_window_count_for_bits)
#define MSM_WINDOWS_MAX (256 / 4 + 1)

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
    long opt_bpt_group = 1;     // basepoint tables: 1 = group a many-table call's items by table before multiplying, 0 = per-lane gathers
    long opt_each_comb = 1;     // verify_each: 1 = per-key comb tables when every key signs >= 8 signatures on average, 2 = always, 0 = never
    long opt_small_straus = 1;  // fewer than 190 pairs: vartime Straus (3 launches) instead of the bucket pipeline
    long opt_field_f64 = 1;     // bucket kernel on the FP64 pipe (fe64.cuh) instead of IMAD.WIDE (fe.cuh)
    // timing of the dominant kernel in the last call
    float last_kernel_ms = 0.f;
    float last_call_ms = 0.f;
    int last_kernel_launches = 0;
    bool async_open = false;       // a ..._partial_async call is in flight: its device span ends in ..._combine_dev
    DevBuf ws[WS_COUNT];            // device workspaces, one per role (WsRole)
    uint32_t hash_seed[4] = {0x243F6A88u, 0x85A308D3u, 0x13198A2Eu, 0x03707344u};   // key of the public-key de-duplication hash, redrawn per context
    int sum_desc_c = -1;
    bool base_table_ready = false;
    bool each_attr_set = false;     // the same for k_verify_each_comb
    bool comb_attr_set = false;     // cudaFuncAttributeMaxDynamicSharedMemorySize set for the comb kernel on this device
    bool sort_attr_set = false;     // the same for the two digit-sort kernels of msm.cu, at their call-independent bounds
    bool comb_base_table_ready = false;
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

#if defined(__CUDACC__)
// *bad |= some thread of the warp had a bad input (good = 0): one warp-wide OR and one atomic per warp, whatever the
// inputs (point_ops.cu, scalars.cu)
__device__ __forceinline__ void warp_report_bad(uint32_t good, int *bad)
{
    const unsigned act = __activemask();
    const uint32_t any_bad = __reduce_or_sync(act, 1u - good);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicOr(bad, (int)any_bad);
}
#endif
// WS_FLAGS, WS_MSM_WINDOWS and WS_MSM_RESULT at their bounds (api.cu): every call that uses them reserves them here
int msm_driver_ws_reserve(dalek_b200_ctx *ctx);
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
// launches on the given stream, with the context's WS_PREP_PROD workspace);
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

// EdwardsPoint::compress_batch (codecs.cu): n extended points as canonical radix-2^51 limbs (device) -> n x 32 B at d_out,
// one shared inversion per CODEC_K points, enqueued on st
void edwards_compress_enqueue(const uint64_t *d_limbs, size_t n, uint32_t *d_out, cudaStream_t st);

// RistrettoPoint::compress of an MSM result (straus.cu): 8 words at d_enc
int ristretto_encode_result(dalek_b200_ctx *ctx, const MsmResult *d_res, uint32_t *d_enc);
