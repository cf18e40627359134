/*
 * dalek_b200.h -- C ABI of the H100 multiscalar-multiplication / batch-verification engine.
 *
 * The reference (curve25519-dalek / ed25519-dalek, 100 % Rust) has no FFI for this path: the
 * hot path sits behind Rust traits.  Each entry point below replaces one of those trait
 * methods / functions and names it (paths relative to the reference tree):
 *
 *   C/ = curve25519-dalek/src/   E/ = ed25519-dalek/src/
 *
 * A thin Rust shim (shown in INTEGRATION.md) collects the trait iterators into the flat
 * buffers used here.  All buffers are caller-owned; unless a `_dev` variant is named, pointers
 * are HOST pointers and the call copies them to the device, runs, copies the result back and
 * returns (blocking).  A context may be used by one thread at a time; different contexts may
 * be used concurrently.
 *
 * Data formats
 *   scalar            32 bytes little-endian, any value < 2^256 (the reference's Scalar
 *                     invariant is bit 255 clear, C/scalar.rs:193-230; not required here)
 *   compressed point  32 bytes CompressedEdwardsY (C/edwards.rs:175) or CompressedRistretto
 *   extended point    20 x uint64_t: X, Y, Z, T as FieldElement51 radix-2^51 limbs
 *                     (C/edwards.rs:390-395, C/backend/serial/u64/field.rs:43); limbs < 2^54
 *
 * Return codes: 0 = success / Ok; positive = the reference's own error values (see the
 * DALEK_* constants); negative = engine errors (bad argument, CUDA failure).  There is no CPU
 * fallback: without a usable CUDA device dalek_b200_init fails with DALEK_E_NO_DEVICE.
 */
#ifndef DALEK_B200_H
#define DALEK_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dalek_b200_ctx dalek_b200_ctx;

/* reference-level outcomes */
#define DALEK_OK 0
#define DALEK_NONE 1                      /* Option::None: a point failed to decompress (C/traits.rs:196) */
#define ED25519_ERR_VERIFY 1              /* InternalError::Verify             (E/errors.rs:38) */
#define ED25519_ERR_ARRAY_LENGTH 2        /* InternalError::ArrayLength        (E/errors.rs:41-49) */
#define ED25519_ERR_SCALAR_FORMAT 3       /* InternalError::ScalarFormat       (E/errors.rs:27) */
#define ED25519_ERR_POINT_DECOMPRESSION 4 /* InternalError::PointDecompression (E/errors.rs:26) */
#define ED25519_ERR_PREHASHED_CONTEXT_LENGTH 5 /* InternalError::PrehashedContextLength (E/errors.rs:50) */
#define ED25519_ERR_MISMATCHED_KEYPAIR 6  /* InternalError::MismatchedKeypair  (E/errors.rs:52) */
/* engine errors */
#define DALEK_E_INVALID_ARG (-1)
#define DALEK_E_NO_DEVICE (-2)
#define DALEK_E_CUDA (-3)
#define DALEK_E_NOMEM (-4)

#define DALEK_POINTS_COMPRESSED 0         /* n x 32 B CompressedEdwardsY */
#define DALEK_POINTS_EXTENDED 1           /* n x 20 x u64 radix-2^51 limbs */
#define DALEK_POINTS_RISTRETTO 2          /* n x 32 B CompressedRistretto (precomputation API and variable-base multiplication) */
#define DALEK_POINTS_MONTGOMERY 3         /* n x 32 B MontgomeryPoint u, canonical (output of dalek_b200_mul_base_ct_batch only) */

/* -------- context ---------------------------------------------------------------------- */
/* Create an engine context on CUDA device `device`.  Fails (no CPU fallback) if the device
 * is missing or is not an sm_90 part (H100). */
int dalek_b200_init(int device, dalek_b200_ctx **out);
void dalek_b200_destroy(dalek_b200_ctx *ctx);
const char *dalek_b200_last_error(const dalek_b200_ctx *ctx);
/* Tunables.  None changes a result except "verify_chunk" (see verify_batch): "window_bits" (4..20, 0 = choose from n),
 * "verify_chunk" (0, default: the reference's single transcript per batch; k > 0: opt-in, one transcript per k signatures --
 * NOT reference-equivalent on inputs with small-order components), "field_f64" (1 = bucket kernel on the FP64-pipe field,
 * default; 0 = IMAD.WIDE field), "acc_tma" (1 = the bucket kernel gathers points with TMA bulk copies, default 0: cp.async),
 * "small_straus" (1 = fewer than 190 pairs run vartime Straus like the reference, default; 0 = bucket pipeline),
 * "host_chunks" (1..8, host-buffer MSM calls stream their input in this many chunks, default 8), "verify_pieces" (1..8, same
 * for verify_batch, default 4), "decompress_f64" (1 = square-root exponentiation of decompression on the FP64 field, default),
 * "dedupe_keys" (1 = decompress every distinct public key once and give it one MSM term, default), "double_base_comb" (1 =
 * fixed-base comb for double-base batches of >= 4096 pairs, default), "precomp_tables" (1 = precomputations of >= 4096 points
 * also keep the 2^(cw) P window tables; default 0: measured, the 1.7 GB of randomly gathered table entries cost the bucket
 * kernel what the shorter tail saves), "transcript_warp" (1 = launches of up to 2048 Merlin transcripts run one warp each,
 * default), "transcript_blocks" (1 = larger launches run one thread per transcript with the rate block staged in shared
 * memory, default; 0 = byte-wise sponge), "each_comb" (per-signature verification: 1 = per-key comb tables when
 * every distinct key signs at least eight signatures on average, default; 2 = always; 0 = never), "bpt_group" (basepoint
 * tables: 1 = a many-table multiplication first groups its items by table on the device, default; 0 = every lane reads its
 * own table), "trace" (1 = per-stage
 * device timeline of verify_batch on stderr).
 * Returns 0 or DALEK_E_INVALID_ARG. */
int dalek_b200_set_option(dalek_b200_ctx *ctx, const char *name, long value);
/* The current value of a tunable named as for dalek_b200_set_option, in *value.  Returns 0 or DALEK_E_INVALID_ARG. */
int dalek_b200_get_option(const dalek_b200_ctx *ctx, const char *name, long *value);
/* Number of kernels launched by this context since creation (bench.py's gpu_launches). */
uint64_t dalek_b200_launch_count(const dalek_b200_ctx *ctx);
/* Milliseconds (CUDA events on the context's stream) spent in the dominant kernel of the last
 * call (bucket accumulation for MSM calls), and that kernel's launch count in the last call. */
int dalek_b200_last_kernel_ms(const dalek_b200_ctx *ctx, float *ms, int *launches);
/* Same by name: "bucket_accumulate" (the figure above) or "decompress_R" (the R-decompression kernel of the last
 * verify_batch call, the largest kernel of that path; summed over the pieces of a host-streamed call). */
int dalek_b200_last_stage_ms(const dalek_b200_ctx *ctx, const char *stage, float *ms);
/* Milliseconds between CUDA events recorded on the context's stream at entry of the last MSM / verify_batch /
 * precomputed-MSM / X25519 / to_montgomery_batch / hash-to-group / Lizard / map_to_curve / map_to_curve_inverse / mul_batch
 * / vartime_double_base_batch / MontgomeryPoint / mul_base_ct_batch / scalar_binary_batch / scalar_unary_batch /
 * scalar_from_bytes_batch / scalar_hash_from_bytes_batch / scalar_fold_batch call, or of the last ed25519_b200_verifying_keys /
 * sign_flat / sign_prehashed / verify_prehashed_each / key_set_new / key_set_verify_flat / key_set_verify_flat_dev /
 * key_set_verify_prehashed / expanded_verifying_keys / raw_sign_flat / raw_sign_prehashed / signing_key_set_new /
 * signing_key_set_sign_flat / signing_key_set_sign_flat_dev / signing_key_set_sign_prehashed call, and after the last work it enqueued (all of the call's streams
 * joined): the device time of that call, copies of host-buffer calls included. */
int dalek_b200_last_call_ms(const dalek_b200_ctx *ctx, float *ms);

/* -------- EdwardsPoint multiscalar multiplication --------------------------------------- */
/*
 * VartimeMultiscalarMul::optional_multiscalar_mul / vartime_multiscalar_mul for EdwardsPoint
 * (C/traits.rs:196-262, C/edwards.rs:1002-1030; algorithms C/backend/serial/scalar_mul/
 * pippenger.rs:67-160 and straus.rs:159-200).  Computes sum scalars[i] * points[i].
 * Returns DALEK_NONE when point_fmt is COMPRESSED and any point fails to decompress
 * (the reference returns None when any Option<Point> is None).  n = 0 yields the identity.
 * out_compressed receives the 32-byte CompressedEdwardsY of the result (EdwardsPoint::compress,
 * C/edwards.rs:564-617); out_limbs (nullable) receives canonical radix-2^51 X,Y,Z,T limbs of an
 * equal point (projectively equal to the reference's result; limb values themselves differ
 * between the reference's own backends).
 */
int dalek_b200_edwards_vartime_msm(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points,
                                   int point_fmt, size_t n, uint8_t out_compressed[32],
                                   uint64_t out_limbs[20]);
/*
 * MultiscalarMul::multiscalar_mul for EdwardsPoint (constant-time contract, C/traits.rs:78-134,
 * C/edwards.rs:970-995, straus.rs:103-144): uniform control flow and table scans that do not
 * depend on the scalars.  Points must all be valid (the trait takes points, not Options):
 * an undecodable compressed point is DALEK_E_INVALID_ARG.
 */
int dalek_b200_edwards_ct_msm(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points,
                              int point_fmt, size_t n, uint8_t out_compressed[32],
                              uint64_t out_limbs[20]);
/* Same two calls with device-resident inputs (scalars: n x 32 B; points as point_fmt says);
 * outputs are still written to host memory. */
int dalek_b200_edwards_vartime_msm_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points,
                                       int point_fmt, size_t n, uint8_t out_compressed[32],
                                       uint64_t out_limbs[20]);

/* -------- sharded MSM (one call per GPU / rank, SURVEY 8e) --------------------------------
 * MSM is linear: every rank reduces a contiguous shard of the pairs to one accumulator per bucket window
 * (pippenger.rs:146-151 for its shard), the accumulators are exchanged once (all-gather: point addition is
 * not an NCCL reduction operator), and every rank adds them per window and runs the Horner pass of
 * pippenger.rs:159.  `n_shard` is the size of the LARGEST shard (ceil(n_total / ranks) for an even split)
 * and must be the same on every rank: the window width is chosen from it, i.e. for the work one GPU does.
 *
 * Number of window accumulators of a partial MSM for that shard size. */
int dalek_b200_msm_window_count(dalek_b200_ctx *ctx, size_t n_shard);
/* Size in bytes of a shard's device RECORD: window_count x 20 u64 limbs, then one u64 status word
 * (non-zero: a compressed point of the shard did not decode -> the combined result is None). */
size_t dalek_b200_msm_partial_bytes(dalek_b200_ctx *ctx, size_t n_shard);
/* Partial MSM over this rank's shard, blocking: writes `window_count` window accumulators
 * (each 20 x u64 extended limbs, window 0 = least significant) to out_windows (host).
 * DALEK_NONE if a compressed point did not decode. */
int dalek_b200_edwards_msm_partial(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points,
                                   int point_fmt, size_t n_local, size_t n_shard,
                                   uint64_t *out_windows);
int dalek_b200_edwards_msm_partial_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points,
                                       int point_fmt, size_t n_local, size_t n_shard,
                                       uint64_t *out_windows);
/* Combine the gathered accumulators of `ranks` shards (host, rank-major: ranks x window_count x 20 u64)
 * into the final point: per-window sum over ranks, then total = total * 2^w + window
 * (pippenger.rs:159). */
int dalek_b200_edwards_msm_combine(dalek_b200_ctx *ctx, const uint64_t *windows, int ranks,
                                   size_t n_shard, uint8_t out_compressed[32], uint64_t out_limbs[20]);
/* The same exchange without leaving the device: ..._partial[_dev]_async ENQUEUES the shard's MSM on the
 * context's stream and writes its record (dalek_b200_msm_partial_bytes) to the device buffer d_out_record;
 * it returns without synchronising.  The caller enqueues the all-gather of the records behind it ON THAT
 * STREAM (dalek_b200_stream: e.g. torch.cuda.ExternalStream + torch.distributed.all_gather_into_tensor, or
 * ncclAllGather(..., stream)), then ..._combine_dev takes the gathered device buffer (ranks records,
 * rank-major), runs the Horner pass and blocks only for the 192-byte result.  DALEK_NONE if any shard's
 * status word is set.  dalek_b200_last_call_ms then spans partial + exchange + combine on the device. */
int dalek_b200_edwards_msm_partial_async(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points,
                                         int point_fmt, size_t n_local, size_t n_shard, void *d_out_record);
int dalek_b200_edwards_msm_partial_dev_async(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points,
                                             int point_fmt, size_t n_local, size_t n_shard, void *d_out_record);
int dalek_b200_edwards_msm_combine_dev(dalek_b200_ctx *ctx, const void *d_records, int ranks, size_t n_shard,
                                       uint8_t out_compressed[32], uint64_t out_limbs[20]);
/* The context's main CUDA stream (a cudaStream_t) for callers that order their own work with the engine's. */
void *dalek_b200_stream(dalek_b200_ctx *ctx);

/* -------- one MSM over several GPUs from a single process (SURVEY 8b / 8e) ---------------------
 * dalek_b200_init_multi creates one engine context per listed CUDA device (distinct sm_90 devices of one node)
 * and enables peer access to the first one.  ..._vartime_msm_multi is VartimeMultiscalarMul::optional_multiscalar_mul
 * (C/traits.rs:196-262, same conventions as dalek_b200_edwards_vartime_msm, host buffers) with the pair range cut
 * into contiguous shards, one per device: every device reduces its shard to window accumulators, the ~2.7 KB records
 * are written into the first device's memory by peer copies over NVLink, and the first device combines them
 * (pippenger.rs:146-159).  Inputs of fewer than 2^14 pairs per device run on the first device alone. */
typedef struct dalek_b200_multi dalek_b200_multi;
int dalek_b200_init_multi(const int *devices, int ndev, dalek_b200_multi **out);
void dalek_b200_destroy_multi(dalek_b200_multi *m);
int dalek_b200_multi_device_count(const dalek_b200_multi *m);
/* The context of device i (e.g. to set options, or to run replicas of verify_batch on every GPU). */
dalek_b200_ctx *dalek_b200_multi_ctx(dalek_b200_multi *m, int i);
const char *dalek_b200_multi_last_error(const dalek_b200_multi *m);
int dalek_b200_edwards_vartime_msm_multi(dalek_b200_multi *m, const uint8_t *scalars, const void *points,
                                         int point_fmt, size_t n, uint8_t out_compressed[32],
                                         uint64_t out_limbs[20]);

/* -------- VartimePrecomputedMultiscalarMul (SURVEY 8f rank 1) ---------------------------------
 * C/traits.rs:290-406; VartimeEdwardsPrecomputation C/edwards.rs:1038-1076, VartimeRistrettoPrecomputation
 * C/ristretto.rs:1004-1049 (serial backend: precomputed_straus.rs:33-127).  The static points are decoded
 * and converted once and stay resident in device memory; later calls send scalars only.  With the option
 * "precomp_tables" the tables 2^(c w) P_i of every window are kept too (96 B x windows per point, e.g. 1.7 GB for
 * 2^20 points), so that all windows share one bucket set and the final doublings disappear.
 *
 * new (traits.rs:297-300): static_points in format DALEK_POINTS_* (RISTRETTO makes a Ristretto
 * precomputation: Ristretto encodings in and out).  DALEK_NONE if an encoded static point does not decode. */
typedef struct dalek_b200_precomp dalek_b200_precomp;
int dalek_b200_precomp_new(dalek_b200_ctx *ctx, const void *static_points, int point_fmt, size_t n,
                           dalek_b200_precomp **out);
size_t dalek_b200_precomp_len(const dalek_b200_precomp *pre);     /* traits.rs:303 */
void dalek_b200_precomp_destroy(dalek_b200_precomp *pre);
/* optional_mixed_multiscalar_mul (traits.rs:402-413):  Q = sum a_i A_i + sum b_j B_j  with B_j the static
 * points.  n_static may be smaller than len() (unused points are ignored, traits.rs:314-316); larger is
 * DALEK_E_INVALID_ARG (the reference asserts).  n_dynamic = 0 gives vartime_multiscalar_mul
 * (traits.rs:324-338).  DALEK_NONE if a dynamic point does not decode.  dynamic_fmt: EXTENDED, or the
 * encoding matching the precomputation (COMPRESSED for Edwards, RISTRETTO for Ristretto).
 * out_compressed: CompressedEdwardsY, or CompressedRistretto for a Ristretto precomputation. */
int dalek_b200_precomp_mixed_msm(dalek_b200_ctx *ctx, const dalek_b200_precomp *pre,
                                 const uint8_t *static_scalars, size_t n_static,
                                 const uint8_t *dynamic_scalars, const void *dynamic_points,
                                 int dynamic_fmt, size_t n_dynamic, uint8_t out_compressed[32],
                                 uint64_t out_limbs[20]);

/* -------- BasepointTable: resident fixed-base tables of any points ------------------------------------------------------
 * C/traits.rs:50-74; EdwardsBasepointTable C/edwards.rs:1127-1243, RistrettoBasepointTable C/ristretto.rs:1080-1115.
 * A handle holds the comb tables of k points P_0..P_{k-1} in device memory: 64 rows of 8 entries (j+1) 16^i P as FP64
 * affine Niels, 61,440 bytes per point, allocated by new and freed by destroy.  The tables are not a context workspace;
 * a handle serves only the context that made it (another context is DALEK_E_INVALID_ARG).
 *   Formats: COMPRESSED and EXTENDED make Edwards tables (CompressedEdwardsY out), RISTRETTO makes Ristretto tables
 *     (CompressedRistretto out); anything else is DALEK_E_INVALID_ARG.
 *   Constant time in the scalars at every batch size: every table row is scanned in full and the sign is applied
 *     inside the addition.  The points, the indices, k and n are public: a table address depends on an index, never on
 *     a scalar.  Every use of a basepoint table (a generator, a recipient's key, a commitment base) has public bases.
 *
 * create (traits.rs:56) for k >= 1 points (k = 0 is DALEK_E_INVALID_ARG): *out = the handle.  If a point does not
 * decode, ok[i] = 0 for it (ok: k bytes, nullable; 1 for every other point), *out stays NULL, nothing stays allocated
 * and the call returns DALEK_NONE.  A failed allocation returns DALEK_E_NOMEM with last_error set and no handle. */
typedef struct dalek_b200_basepoint_tables dalek_b200_basepoint_tables;
int dalek_b200_basepoint_tables_new(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t k,
                                    uint8_t *ok /* k bytes, nullable */, dalek_b200_basepoint_tables **out);
size_t dalek_b200_basepoint_tables_len(const dalek_b200_basepoint_tables *t);
/* destroy waits for the device and frees the tables; it does not use the context, so a handle may be destroyed before
 * or after its context.  NULL is a no-op. */
void dalek_b200_basepoint_tables_destroy(dalek_b200_basepoint_tables *t);
/* basepoint (traits.rs:59, C/edwards.rs:1144-1148, C/ristretto.rs:1108-1110): the k encodings of P_i read back from
 * entry (0, 0) of each table: the canonical encoding of the decoded point (a non-canonical CompressedEdwardsY comes
 * back canonical, a Ristretto point as the canonical encoding of its coset). */
int dalek_b200_basepoint_tables_basepoints(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t,
                                           uint8_t *out /* k x 32 B */);
/* mul_base / mul_base_clamped (traits.rs:62-74, C/edwards.rs:1192-1243): out[i] = s_i P_{t_i}, t_i = indices[i]
 * (indices NULL: table 0 serves every item).  The scalar is used as the integer it is, not reduced mod l, so out[i]
 * equals dalek_b200_mul_batch(s_i, P_{t_i}) for every input, points with a torsion component included.  flags = 0:
 * bit 255 set is DALEK_E_INVALID_ARG; flags = DALEK_MUL_CLAMPED: any 32 bytes, clamped (clamp_integer,
 * C/scalar.rs:1407-1412) and not reduced, for Edwards and Ristretto tables alike (the trait's default method).  Other
 * flag bits are DALEK_E_INVALID_ARG.  An index >= k is DALEK_E_INVALID_ARG.  Host buffers: the scalar and index checks
 * run before any device work; the batch is streamed in pieces and the device copies of the scalars and results are
 * cleared before the call returns, failed calls included.  n = 0 is a successful no-op; a NULL scalars or out with
 * n > 0 is DALEK_E_INVALID_ARG.  With indices, the items are first grouped by table on the device (a counting sort of
 * the public indices; option "bpt_group"), so that the threads of a warp read the same table rows. */
int dalek_b200_basepoint_tables_mul(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t,
                                    const uint8_t *scalars, const uint32_t *indices /* n, or NULL */, size_t n,
                                    int flags, uint8_t *out /* n x 32 B */);
/* same, every buffer a device pointer; blocks until done.  A scalar with bit 255 set (without the clamp flag) or an
 * index >= k is reported after the batch ran: the call returns DALEK_E_INVALID_ARG and the outputs are unspecified.
 * An index >= k is never used as an address: the kernel reads table 0 in its place. */
int dalek_b200_basepoint_tables_mul_dev(dalek_b200_ctx *ctx, const dalek_b200_basepoint_tables *t,
                                        const void *d_scalars, const void *d_indices, size_t n, int flags, void *d_out);

/* -------- batch wire-format codecs (SURVEY 8f rank 2) -----------------------------------------
 * Points are the reference's in-memory EdwardsPoint / RistrettoPoint: 20 u64 limbs X | Y | Z | T, radix 2^51.
 * Host buffers; the batch is streamed in pieces so that the copies overlap the arithmetic.
 *
 * CompressedEdwardsY::decompress (C/edwards.rs:211-257) for n encodings: ok[i] = 1 and out_limbs[20 i ..] =
 * the point (Z = 1), or ok[i] = 0 (None; the slot holds the identity).  Returns DALEK_NONE if any ok[i] = 0. */
int dalek_b200_edwards_decompress_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n,
                                        uint64_t *out_limbs, uint8_t *ok);
/* EdwardsPoint::compress_batch (C/edwards.rs:619-647): n points -> n x 32 B, one shared inversion per 8
 * points (FieldElement::invert_batch, C/field.rs:239-274). */
int dalek_b200_edwards_compress_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n, uint8_t *out);
/* CompressedRistretto::decompress (C/ristretto.rs:266-345), same conventions as the Edwards form. */
int dalek_b200_ristretto_decompress_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n,
                                          uint64_t *out_limbs, uint8_t *ok);
/* RistrettoPoint::double_and_compress_batch (C/ristretto.rs:564-646): out[i] = compress(2 P_i). */
int dalek_b200_ristretto_double_and_compress_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n,
                                                   uint8_t *out);
/* EdwardsPoint::to_montgomery_batch (C/edwards.rs:592-612): n x 20 u64 limbs -> n x 32 B Montgomery u = (Z+Y)/(Z-Y),
 * one shared inversion per 8 points; the identity (Z = Y) gives u = 0. */
int dalek_b200_edwards_to_montgomery_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n, uint8_t *out);

/* -------- X25519 (x25519-dalek, RFC 7748) ------------------------------------------------------
 * Scalars are 32-byte secrets, clamped inside the call (clamp_integer, C/scalar.rs:1407-1412) and not reduced; u
 * coordinates are read like FieldElement::from_bytes (bit 255 ignored, values in [p, 2^255) accepted).  Both calls are
 * constant time in the secrets: uniform control flow, XOR-mask swaps, full-row table scans.  Host-buffer calls stream
 * the batch in pieces like the codecs and clear the device copies of the secrets and results before returning.
 * n = 0 is a successful no-op; a NULL buffer with n > 0 is DALEK_E_INVALID_ARG.  The option "field_f64" has no effect.
 *
 * x25519(k_i, u_i) (x25519-dalek x25519.rs:390-392); out: n x 32 B; contributory: n bytes or NULL. Never fails on input values. */
int dalek_b200_x25519_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, const uint8_t *us, size_t n,
                            uint8_t *out, uint8_t *contributory);
/* same, every buffer a device pointer; blocks until done */
int dalek_b200_x25519_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_us, size_t n,
                                void *d_out, void *d_contributory);
/* PublicKey::from(&StaticSecret) = mul_base_clamped(k).to_montgomery(); out: n x 32 B */
int dalek_b200_x25519_public_keys(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, uint8_t *out);

/* -------- MontgomeryPoint (C/montgomery.rs) -------------------------------------------------------
 * u coordinates are 32 bytes read like FieldElement::from_bytes (bit 255 ignored, values in [p, 2^255) accepted, points
 * of the twist accepted); results are canonical.  Broadcast: n_scalars / n_ints and n_points are each 1 or n; 1 uses
 * that input for every item, any other value is DALEK_E_INVALID_ARG.  n = 0 is a successful no-op; a NULL buffer with
 * n > 0 is DALEK_E_INVALID_ARG, except ok.  The ladders are constant time in the scalars / integers and in u: nbits is
 * public, the swaps are XOR masks and no address depends on a bit.  Host-buffer calls stream the batch in pieces like
 * the codecs and clear the device copies of the scalars and results before they return.
 *
 * Scalar * MontgomeryPoint (C/montgomery.rs:484-505): out[i] = u([s_i] P_i), the ladder over bits 254..0 of the
 * unclamped, unreduced Scalar s_i.  A scalar with bit 255 set (Scalar invariant #1) is DALEK_E_INVALID_ARG before any
 * device work.  mul_clamped (montgomery.rs:150-161) is dalek_b200_x25519_batch. */
int dalek_b200_montgomery_mul_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n_scalars, const uint8_t *us,
                                    size_t n_points, size_t n, uint8_t *out /* n x 32 B */);
/* same, every buffer a device pointer; blocks until done.  A scalar with bit 255 set is reported after the batch ran:
 * the call returns DALEK_E_INVALID_ARG and the outputs are unspecified. */
int dalek_b200_montgomery_mul_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, size_t n_scalars, const void *d_us,
                                        size_t n_points, size_t n, void *d_out);
/* MontgomeryPoint::mul_bits_be (C/montgomery.rs:176-211): out[i] = u([b_i] P_i) for the integer b_i given by bits
 * nbits-1..0 of ints[i], an int_bytes-byte little-endian integer (1 <= int_bytes <= 64, 0 <= nbits <= 8 int_bytes;
 * otherwise DALEK_E_INVALID_ARG).  The ladder runs one step per bit from bit nbits-1 down, whatever the bits are;
 * nbits = 0 gives u = 0 (as_affine of the identity, montgomery.rs:409-412).  Any bit values are accepted. */
int dalek_b200_montgomery_mul_bits_be_batch(dalek_b200_ctx *ctx, const uint8_t *ints, size_t int_bytes, size_t n_ints,
                                            size_t nbits, const uint8_t *us, size_t n_points, size_t n,
                                            uint8_t *out /* n x 32 B */);
/* MontgomeryPoint::to_edwards (C/montgomery.rs:223-268): y = (u - 1) / (u + 1), bit 7 of its last byte flipped by bit 0
 * of signs[i] (the u8 shift of the reference), then CompressedEdwardsY::decompress (C/edwards.rs:211-257).  out[i] is
 * the CompressedEdwardsY of the point.  u = -1 (either encoding) and u of the twist are None: ok[i] = 0, the identity's
 * encoding in the slot and the call returns DALEK_NONE; every other ok[i] is 1.  Host buffers, streamed in pieces. */
int dalek_b200_montgomery_to_edwards_batch(dalek_b200_ctx *ctx, const uint8_t *us, const uint8_t *signs /* n bytes */,
                                           size_t n, uint8_t *out /* n x 32 B */, uint8_t *ok /* n bytes, nullable */);

/* -------- constant-time fixed-base scalar multiplication ------------------------------------------
 * out[i] = s_i B, B the Ed25519 basepoint: EdwardsPoint::mul_base / mul_base_clamped (C/edwards.rs:918-957),
 * RistrettoPoint::mul_base (C/ristretto.rs:939) and MontgomeryPoint::mul_base / mul_base_clamped (C/montgomery.rs:143-174,
 * EdwardsPoint::mul_base(s).to_montgomery()).  out_fmt: DALEK_POINTS_COMPRESSED (CompressedEdwardsY),
 * DALEK_POINTS_RISTRETTO (CompressedRistretto) or DALEK_POINTS_MONTGOMERY (u), 32 B each; anything else is
 * DALEK_E_INVALID_ARG.  flags = 0: scalars with bit 255 clear (else DALEK_E_INVALID_ARG), not reduced; as B has order l the
 * point is (s mod l) B.  flags = DALEK_MUL_CLAMPED: any 32 bytes, clamped (clamp_integer, C/scalar.rs:1407-1412); the
 * reference has no RistrettoPoint::mul_base_clamped, so the flag with RISTRETTO is DALEK_E_INVALID_ARG.  Other flag bits
 * are DALEK_E_INVALID_ARG.  n = 0 is a successful no-op; a NULL buffer with n > 0 is DALEK_E_INVALID_ARG.
 * Constant time in the scalars at every batch size: the comb of dalek_b200_x25519_public_keys over the context's cached
 * table of B, every table row scanned in full.  Host buffers, streamed in pieces; the device copies of the scalars and
 * results are cleared before the call returns.  (dalek_b200_edwards_mul_base_batch indexes its table by the digit and is
 * for public scalars only.) */
int dalek_b200_mul_base_ct_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n, int out_fmt, int flags,
                                 uint8_t *out /* n x 32 B */);

/* -------- variable-base scalar multiplication -------------------------------------------------
 * out[i] = s_i * P_i: EdwardsPoint * Scalar (C/edwards.rs:890-899 -> C/backend/serial/scalar_mul/variable_base.rs:11-48),
 * EdwardsPoint::mul_clamped (C/edwards.rs:932-941) and RistrettoPoint * Scalar (C/ristretto.rs:917-926).
 * BasepointTable::create(P) * s, with the table kept between calls, is dalek_b200_basepoint_tables_mul; it gives the
 * same points.
 *   Broadcast: n_scalars and n_points are each 1 or n; 1 uses that input for every item, any other value is
 *     DALEK_E_INVALID_ARG.  n = 0 is a successful no-op.  A NULL buffer with n > 0 is DALEK_E_INVALID_ARG, except ok.
 *   Point formats: COMPRESSED (CompressedEdwardsY in and out), EXTENDED (20 radix-2^51 limbs in, any Z;
 *     CompressedEdwardsY out), RISTRETTO (CompressedRistretto in and out, C/ristretto.rs:500-533).
 *   An undecodable point gives ok[i] = 0 and the identity's encoding in its slot, and the call returns DALEK_NONE, as
 *     dalek_b200_edwards_decompress_batch does; every other ok[i] is 1.
 *   Scalars: 32 bytes little-endian with bit 255 clear (Scalar invariant #1, as in dalek_b200_edwards_ct_msm), else
 *     DALEK_E_INVALID_ARG.  With flags = DALEK_MUL_CLAMPED any 32 bytes are accepted, clamped inside the call
 *     (clamp_integer, C/scalar.rs:1407-1412) and not reduced; the reference has no clamped Ristretto multiplication,
 *     so DALEK_MUL_CLAMPED with RISTRETTO is DALEK_E_INVALID_ARG.  Other flag bits are DALEK_E_INVALID_ARG.
 *   Constant time in the scalars: no branch, loop bound or address depends on them (masked full scans of 8-entry
 *     tables and a masked sign, window.rs:54-76).  Host-buffer calls stream the batch in pieces like the codecs and
 *     clear the device copies of the scalars and of the results before they return.  No option affects these calls. */
#define DALEK_MUL_CLAMPED 1
int dalek_b200_mul_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n_scalars, const void *points, int point_fmt,
                         size_t n_points, size_t n, int flags, uint8_t *out /* n x 32 B */, uint8_t *ok /* n bytes, nullable */);
/* same, every buffer a device pointer; blocks until done.  A scalar with bit 255 set (without the clamp flag) is
 * reported after the batch ran: the call returns DALEK_E_INVALID_ARG and the outputs are unspecified. */
int dalek_b200_mul_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, size_t n_scalars, const void *d_points, int point_fmt,
                             size_t n_points, size_t n, int flags, void *d_out, void *d_ok);
/* out[i] = is_small_order(P_i) | is_torsion_free(P_i) << 1 | decoded << 2 (C/edwards.rs:1405-1437; VerifyingKey::is_weak is
 * is_small_order).  points: COMPRESSED or EXTENDED, anything else is DALEK_E_INVALID_ARG.  An undecodable point gives
 * out[i] = 0; the call still returns DALEK_OK.  Host buffers, streamed in pieces. */
int dalek_b200_edwards_torsion_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n, uint8_t *out);

/* -------- variable-time double-base scalar multiplication ----------------------------------------
 * EdwardsPoint::vartime_double_scalar_mul_basepoint (C/edwards.rs:1078-1087 -> vartime_double_base.rs:23-72) and
 * RistrettoPoint::vartime_double_scalar_mul_basepoint (C/ristretto.rs:1051-1063): out[i] = a_i A_i + b_i B, B the
 * Ed25519 (= Ristretto) basepoint; the operation of every Schnorr-style verification, R' = [k](-A) + [s]B.
 *   ab holds n pairs a_i || b_i of 32-byte little-endian scalars.  Each must have bit 255 clear (Scalar invariant #1),
 *     else DALEK_E_INVALID_ARG, found before any device work.  Scalars in [l, 2^255) are used as given, not reduced: A_i
 *     may carry a torsion component, and then a A_i != (a mod l) A_i.
 *   Point formats as dalek_b200_mul_batch: COMPRESSED (CompressedEdwardsY in and out), EXTENDED (20 radix-2^51 limbs in,
 *     any Z, limbs < 2^54; CompressedEdwardsY out), RISTRETTO (CompressedRistretto in and out); any other point_fmt is
 *     DALEK_E_INVALID_ARG.  An undecodable point gives ok[i] = 0 and the identity's encoding in its slot, and the call
 *     returns DALEK_NONE; every other slot is computed and its ok[i] is 1.
 *   n = 0 is a successful no-op.  A NULL ab, points or out with n > 0 is DALEK_E_INVALID_ARG; ok may be NULL.
 *   Variable time: scalars and points are public, so nothing is cleared.  Host buffers are streamed in pieces like the
 *     codecs.  No option affects these calls. */
int dalek_b200_vartime_double_base_batch(dalek_b200_ctx *ctx, const uint8_t *ab /* n x 64 B: a_i || b_i */,
                                         const void *points, int point_fmt, size_t n,
                                         uint8_t *out /* n x 32 B */, uint8_t *ok /* n bytes, nullable */);
/* same, every buffer a device pointer; blocks until done.  A scalar with bit 255 set is reported after the batch ran:
 * the call returns DALEK_E_INVALID_ARG and the outputs are unspecified. */
int dalek_b200_vartime_double_base_batch_dev(dalek_b200_ctx *ctx, const void *d_ab, const void *d_points, int point_fmt,
                                             size_t n, void *d_out, void *d_ok);

/* -------- many independent MSMs in one call ----------------------------------------------------
 * m multiscalar multiplications, each with its own scalars and its own points: MSM j is the sum of s_i * P_i over the
 * terms offsets[j] <= i < offsets[j+1] of the flat arrays, and out holds one result per MSM.  Per MSM the semantics are
 * those of the single calls on its segment:
 *   constant_time = 0: VartimeMultiscalarMul::optional_multiscalar_mul (C/traits.rs:196-262, C/edwards.rs:1002-1030,
 *     C/ristretto.rs:979-994).  An undecodable point makes that MSM None: ok[j] = 0, its slot holds the identity's
 *     encoding (and limbs), every other MSM is unaffected and the call returns DALEK_NONE; otherwise DALEK_OK.
 *   constant_time = 1: MultiscalarMul::multiscalar_mul (C/traits.rs:78-134, C/edwards.rs:970-995,
 *     C/backend/serial/scalar_mul/straus.rs:103-144; for RISTRETTO C/ristretto.rs:964-977): no branch, loop bound or
 *     address depends on a scalar; the segment sizes and the points are public.  An undecodable point is
 *     DALEK_E_INVALID_ARG for the call (ok still says where), and so is a scalar with bit 255 set (Scalar invariant #1),
 *     found before any device work.  The device copies of the scalars, their digits, the per-term tables and the
 *     partial sums are cleared before the call returns.
 *   offsets: m + 1 values, offsets[0] = 0, non-decreasing, offsets[m] = total < 2^31, else DALEK_E_INVALID_ARG before any
 *     device work.  An empty segment gives the identity.  m = 0 is a successful no-op.  A NULL offsets or out with m > 0,
 *     or NULL scalars or points with total > 0, is DALEK_E_INVALID_ARG; out_limbs and ok may be NULL.
 *   Point formats: COMPRESSED and EXTENDED give CompressedEdwardsY results, RISTRETTO gives CompressedRistretto;
 *     out_limbs are canonical radix-2^51 limbs (X | Y | Z | T) of an equal point.
 *   Every result is the group element the single call returns for that segment.  Variable-time scalars are any 256-bit
 *     values, as in dalek_b200_edwards_vartime_msm.  Variable-time segments of 2^15 terms or more run through the
 *     single-MSM pipeline inside the call; the rest of the batch runs in pieces of whole MSMs of at most 2^18 terms on two
 *     streams, about 1.3 KiB of workspace per term of a piece (a constant-time MSM larger than a piece is a piece of its
 *     own).  No option affects these calls. */
int dalek_b200_msm_batch(dalek_b200_ctx *ctx, const uint8_t *scalars /* total x 32 B */, const void *points, int point_fmt,
                         const uint64_t *offsets /* m + 1 */, size_t m, int constant_time, uint8_t *out /* m x 32 B */,
                         uint64_t *out_limbs /* nullable, m x 20 */, uint8_t *ok /* nullable, m bytes */);
/* same with scalars, points and offsets in device memory; the results go to host memory.  The offsets are read back
 * once (8 bytes per MSM) to check them and to size the pieces.  A scalar with bit 255 set in constant-time mode is
 * reported after the batch ran: the call returns DALEK_E_INVALID_ARG and the outputs are unspecified.  The engine's digits,
 * tables and partial sums are cleared as above; the input buffers are the caller's. */
int dalek_b200_msm_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points, int point_fmt, const void *d_offsets,
                             size_t m, int constant_time, uint8_t *out, uint64_t *out_limbs, uint8_t *ok);

/* -------- group operations on Edwards and Ristretto points --------------------------------------
 * Add, Sub, Neg, Group::double, mul_by_cofactor, ct_eq / is_identity and Sum (C/edwards.rs:501-520, :786-876, :1365-1367;
 * C/ristretto.rs:809-908; C/traits.rs:33-48) over batches.
 *   The input format fixes the group: COMPRESSED is Edwards, RISTRETTO is Ristretto, EXTENDED (20 radix-2^51 limbs, any Z)
 *     is Edwards unless flags carry DALEK_POINT_RISTRETTO, which makes the limbs a Ristretto representative.  The flag
 *     with COMPRESSED is DALEK_E_INVALID_ARG.
 *   out_fmt is the group's own encoding (COMPRESSED for Edwards, RISTRETTO for Ristretto) or EXTENDED: canonical limbs of
 *     an equal point (a representative of the coset for Ristretto), so that chains stay on the device without decoding
 *     again.  Any other combination is DALEK_E_INVALID_ARG.
 *   Broadcast: n_a and n_b are each 1 or n.  n = 0 (m = 0) is a successful no-op.  A NULL buffer with items to process is
 *     DALEK_E_INVALID_ARG, except ok.  Bad formats, flags, ops and offsets are found before any device work.
 *   An undecodable input gives ok[i] = 0 and the identity's encoding (or limbs) in its slot, and the call returns
 *     DALEK_NONE; every other ok[i] is 1.
 *   Constant time in the points: no branch, loop bound or address depends on a coordinate, a decode outcome or an
 *     equality; counts, offsets, formats, ops and flags are public.  Host-buffer calls stream the batch in pieces and
 *     clear the device copies of their inputs, intermediates and results before they return, also after a failed
 *     launch; the _dev calls clear the engine's intermediates.  No option affects these calls. */
#define DALEK_POINT_SUB 1                 /* point_add_batch: out = A - B */
#define DALEK_POINT_RISTRETTO 2           /* EXTENDED points are Ristretto representatives */
#define DALEK_POINT_NEG 0                 /* point_unary_batch ops */
#define DALEK_POINT_DOUBLE 1
#define DALEK_POINT_MUL_BY_COFACTOR 2     /* Edwards only: a Ristretto input is DALEK_E_INVALID_ARG */
/* out[i] = A_i + B_i, or A_i - B_i with DALEK_POINT_SUB.  out: n x 32 B, or n x 160 B for EXTENDED. */
int dalek_b200_point_add_batch(dalek_b200_ctx *ctx, const void *a, size_t n_a, const void *b, size_t n_b, int in_fmt, size_t n,
                               int flags, int out_fmt, void *out, uint8_t *ok /* n bytes, nullable */);
/* same, every buffer a device pointer; blocks until done */
int dalek_b200_point_add_batch_dev(dalek_b200_ctx *ctx, const void *d_a, size_t n_a, const void *d_b, size_t n_b, int in_fmt,
                                   size_t n, int flags, int out_fmt, void *d_out, void *d_ok);
/* out[i] = -P_i, 2 P_i or 8 P_i (op DALEK_POINT_NEG, _DOUBLE, _MUL_BY_COFACTOR); any other op is DALEK_E_INVALID_ARG */
int dalek_b200_point_unary_batch(dalek_b200_ctx *ctx, int op, const void *points, int in_fmt, size_t n, int flags, int out_fmt,
                                 void *out, uint8_t *ok);
int dalek_b200_point_unary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_points, int in_fmt, size_t n, int flags,
                                     int out_fmt, void *d_out, void *d_ok);
/* out[i] = eq | both_decoded << 1, eq the group's ct_eq (Edwards: X1 Z2 = X2 Z1 and Y1 Z2 = Y2 Z1; Ristretto:
 * X1 Y2 = Y1 X2 or X1 X2 = Y1 Y2), 0 when an input does not decode (the call then returns DALEK_NONE).  b = NULL compares
 * with the identity (is_identity; n_b is ignored).  Points are compared as group elements, not as bytes: a non-canonical
 * CompressedEdwardsY equals its canonical form, and two representatives of one Ristretto coset are equal as Ristretto
 * points and unequal as Edwards points.  Host buffers. */
int dalek_b200_point_eq_batch(dalek_b200_ctx *ctx, const void *a, size_t n_a, const void *b, size_t n_b, int in_fmt, size_t n,
                              int flags, uint8_t *out /* n bytes */);
/* Sum (fold from the identity) of each segment: result j is the sum of the points offsets[j] .. offsets[j+1] (m + 1 u64
 * offsets, offsets[0] = 0, non-decreasing, offsets[m] < 2^31, else DALEK_E_INVALID_ARG before any device work).  An empty
 * segment gives the identity; a segment with an undecodable point gives ok[j] = 0 and the identity.  out: m x 32 B, or
 * m x 160 B for EXTENDED. */
int dalek_b200_point_sum_batch(dalek_b200_ctx *ctx, const void *points, int in_fmt, int flags, const uint64_t *offsets, size_t m,
                               int out_fmt, void *out, uint8_t *ok /* m bytes, nullable */);
/* same, every buffer a device pointer; the offsets are read back once (8 bytes per segment) to plan the chunks */
int dalek_b200_point_sum_batch_dev(dalek_b200_ctx *ctx, const void *d_points, int in_fmt, int flags, const void *d_offsets, size_t m,
                                   int out_fmt, void *d_out, void *d_ok);

/* -------- hash to group ------------------------------------------------------------------------
 * Host buffers; each call blocks and streams the batch in pieces like the codecs.  The maps are total: these calls never
 * return DALEK_NONE.  n = 0 is a successful no-op; with n > 0 a NULL buffer other than msgs_flat is DALEK_E_INVALID_ARG.
 * Flat messages, the layout of every host-buffer call that takes msgs_flat and msg_offsets: message i =
 * msgs_flat[msg_offsets[i] .. msg_offsets[i+1]) (n + 1 offsets).  For n > 0, msg_offsets must not be NULL,
 * msg_offsets[0] must be 0, the offsets must not decrease, and msgs_flat may be NULL only when every message is empty
 * (msg_offsets[n] = 0); otherwise the call returns DALEK_E_INVALID_ARG.  Constant time in the message bytes (only the
 * lengths of the messages and of the DST shape the work).  No option affects these calls.
 *
 * RistrettoPoint::from_uniform_bytes (C/ristretto.rs:774-790): in n x 64 B -> out n x 32 B CompressedRistretto */
int dalek_b200_ristretto_from_uniform_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out);
/* RistrettoPoint::hash_from_bytes::<Sha512> (C/ristretto.rs:736-761): out n x 32 B CompressedRistretto */
int dalek_b200_ristretto_hash_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                               size_t n, uint8_t *out);
/* EdwardsPoint::hash_to_curve::<Sha512> (C/edwards.rs:736-750, RFC 9380 edwards25519_XMD:SHA-512_ELL2_RO_) and
 * EdwardsPoint::encode_to_curve::<Sha512> (C/edwards.rs:710-721, ..._ELL2_NU_): one DST of 1..255 bytes for the whole batch
 * (dst_len 0 or > 255 is DALEK_E_INVALID_ARG, where the reference panics, C/field.rs:457-462); out n x 32 B
 * CompressedEdwardsY */
int dalek_b200_edwards_hash_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                           size_t n, const uint8_t *dst, size_t dst_len, uint8_t *out);
int dalek_b200_edwards_encode_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                             size_t n, const uint8_t *dst, size_t dst_len, uint8_t *out);

/* -------- Lizard and the Elligator inverse ------------------------------------------------------
 * Lizard (C/lizard/) is an injective map from 16-byte strings into ristretto255, for ElGamal encryption of short payloads.
 * Host buffers; each call blocks and streams the batch in pieces like hash to group.  n = 0 is a successful no-op; with
 * n > 0 a NULL buffer is DALEK_E_INVALID_ARG.  No option affects these calls.  The digest is fixed to SHA-256 (the
 * reference is generic over any 32-byte Digest and says "Use SHA-256 if otherwise unsure").  Points are
 * DALEK_POINTS_RISTRETTO (CompressedRistretto) or DALEK_POINTS_EXTENDED (20 radix-2^51 limbs, any Z, trusted to be a valid
 * RistrettoPoint representative and used exactly as given: the candidate order of the inverse depends on the
 * representative); any other point_fmt is DALEK_E_INVALID_ARG.  Constant time in the payloads, the points and the
 * recovered payloads.  Every call clears the device copies of its staged inputs and outputs before it returns.
 * map_to_curve_restricted is map_to_curve with a precondition assertion and has no entry point of its own.
 *
 * RistrettoPoint::map_to_curve (C/ristretto/elligator.rs:62-67): n x 32 B -> n x 32 B CompressedRistretto; bit 255 ignored. */
int dalek_b200_ristretto_map_to_curve_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out);
/* RistrettoPoint::lizard_encode::<Sha256> (C/lizard/lizard_ristretto.rs:25-39): n x 16 B -> n x 32 B CompressedRistretto. */
int dalek_b200_ristretto_lizard_encode_batch(dalek_b200_ctx *ctx, const uint8_t *data, size_t n, uint8_t *out);
/* RistrettoPoint::lizard_decode::<Sha256> (:43-71).  data_out n x 16 B, status n bytes: 0 = Some (payload in data_out),
 * 1 = None (a point, but not exactly one candidate passes), 2 = encoding does not decode.  Slots with status != 0 hold
 * zeros.  Returns DALEK_OK if every status is 0, else DALEK_NONE. */
int dalek_b200_ristretto_lizard_decode_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n,
                                             uint8_t *data_out, uint8_t *status);
/* RistrettoPoint::map_to_curve_inverse (:213-219).  out n x 16 x 32 B: candidate j of item i at out[512 i + 32 j], in the
 * reference's order (jc0, dual(jc0), ..., jc3, dual(jc3), then their negations); zero bytes where None.  mask n x u16:
 * bit j set iff candidate j is Some.  An undecodable encoding gives mask 0 and makes the call return DALEK_NONE. */
int dalek_b200_ristretto_map_to_curve_inverse_batch(dalek_b200_ctx *ctx, const void *points, int point_fmt, size_t n,
                                                    uint8_t *out, uint16_t *mask);

/* -------- scalar batch helpers (SURVEY 8f rank 4) ---------------------------------------------
 * Scalar::from_bytes_mod_order_wide (C/scalar.rs:248-250) for n 64-byte strings -> n canonical 32-byte scalars. */
int dalek_b200_scalar_from_wide_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out);
/* Scalar::invert_batch / invert_batch_alloc (C/scalar.rs:779-853): out[i] = in[i]^-1 mod l (inputs are taken mod l),
 * out_product = the product of all inverses (the reference's return value; 1 for n = 0).  The reference requires
 * nonzero inputs (scalar.rs:796-799): a zero input is DALEK_E_INVALID_ARG here. */
int dalek_b200_scalar_invert_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out,
                                   uint8_t out_product[32]);

/* -------- scalar arithmetic ------------------------------------------------------------------------
 * Add, Sub, Mul, Neg, invert, div_by_2, from_bytes_mod_order, from_canonical_bytes, hash_from_bytes, Sum and Product of
 * Scalar (C/scalar.rs:235-263, :317-374, :454-476, :617-670, :739-741, :858-870) over batches of 32-byte little-endian
 * scalars.
 *   Inputs of the arithmetic (binary, unary and fold calls) must be canonical, < l (Scalar invariant #2,
 *     C/scalar.rs:207-228).  Bit 255 set or a value in [l, 2^255) makes the call return DALEK_E_INVALID_ARG after the
 *     batch has run, host and _dev calls alike; the outputs are then unspecified.  Inputs are never reduced silently:
 *     the reference's own Add and Sub are wrong for unreduced scalars (clamped secrets, for example).
 *   Results are canonical.  invert(0) = 0 (the reference's exponentiation gives 0^(l-2) = 0), Neg(0) = 0, the empty Sum
 *     is 0 and the empty Product is 1.
 *   Broadcast: n_a and n_b are each 1 or n.  out may equal a non-broadcast input exactly (in place); any other overlap is
 *     the caller's error.  n = 0 (m = 0) is a successful no-op.  A NULL buffer with items to process is
 *     DALEK_E_INVALID_ARG, except ok.  Bad ops, modes and offsets, and item counts of 2^56 or more, are found before any device
 *     work.
 *   Constant time in the scalar values at every batch size: no branch, loop bound or address depends on a value; the op,
 *     mode, counts, broadcast and segment offsets are public, and so is the inversion's exponent l - 2.
 *   Host-buffer calls stream the batch in pieces and clear the device copies of their inputs, intermediates and results
 *     before they return, also after a failed launch; the _dev calls clear the engine's intermediates.  No option affects
 *     these calls. */
#define DALEK_SCALAR_ADD 0                /* scalar_binary_batch ops */
#define DALEK_SCALAR_SUB 1
#define DALEK_SCALAR_MUL 2
#define DALEK_SCALAR_NEG 0                /* scalar_unary_batch ops */
#define DALEK_SCALAR_INVERT 1             /* Scalar::invert per item; 0 -> 0 */
#define DALEK_SCALAR_DIV_BY_2 2
#define DALEK_SCALAR_SUM 0                /* scalar_fold_batch ops */
#define DALEK_SCALAR_PRODUCT 1
#define DALEK_SCALAR_MOD_ORDER 0          /* scalar_from_bytes_batch modes */
#define DALEK_SCALAR_CANONICAL 1
/* out[i] = A_i + B_i, A_i - B_i or A_i * B_i (op DALEK_SCALAR_ADD, _SUB, _MUL).  out: n x 32 B. */
int dalek_b200_scalar_binary_batch(dalek_b200_ctx *ctx, int op, const uint8_t *a, size_t n_a, const uint8_t *b, size_t n_b, size_t n,
                                   uint8_t *out);
/* same, every buffer a device pointer; blocks until done */
int dalek_b200_scalar_binary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_a, size_t n_a, const void *d_b, size_t n_b, size_t n,
                                       void *d_out);
/* out[i] = -S_i, S_i^-1 (0 for 0) or S_i / 2 (op DALEK_SCALAR_NEG, _INVERT, _DIV_BY_2) */
int dalek_b200_scalar_unary_batch(dalek_b200_ctx *ctx, int op, const uint8_t *in, size_t n, uint8_t *out);
int dalek_b200_scalar_unary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_in, size_t n, void *d_out);
/* MOD_ORDER: Scalar::from_bytes_mod_order, any 32 bytes reduced mod l (ok all 1).  CANONICAL:
 * Scalar::from_canonical_bytes, ok[i] = 0 and zero bytes for bit 255 set or value >= l (None); the call then returns
 * DALEK_NONE.  Host buffers; ok n bytes, nullable. */
int dalek_b200_scalar_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, int mode, uint8_t *out, uint8_t *ok);
/* Scalar::hash_from_bytes::<Sha512>: SHA-512 of each message, reduced mod l as from_bytes_mod_order_wide.  Flat messages
 * as in the hash-to-group block; constant time in the message bytes.  out: n x 32 B. */
int dalek_b200_scalar_hash_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n,
                                            uint8_t *out);
/* Sum / Product (op DALEK_SCALAR_SUM, _PRODUCT) of each segment: result j folds the scalars offsets[j] .. offsets[j+1]
 * (m + 1 u64 offsets, offsets[0] = 0, non-decreasing, offsets[m] < 2^31, else DALEK_E_INVALID_ARG before any device
 * work).  out: m x 32 B.  The ring is commutative, so the result is exact whatever order the fold takes. */
int dalek_b200_scalar_fold_batch(dalek_b200_ctx *ctx, int op, const uint8_t *scalars, const uint64_t *offsets, size_t m, uint8_t *out);
/* same, every buffer a device pointer; the offsets are read back once (8 bytes per segment) to plan the chunks */
int dalek_b200_scalar_fold_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_scalars, const void *d_offsets, size_t m, void *d_out);

/* -------- RistrettoPoint ----------------------------------------------------------------- */
/* n independent RistrettoPoint::multiscalar_mul([a_i, b_i], [G, H]) (constant-time Straus,
 * C/ristretto.rs:964-977 -> C/edwards.rs:970-995 -> straus.rs:103-144), each result compressed
 * (RistrettoPoint::compress, C/ristretto.rs:500-533).  G, H: CompressedRistretto; a, b: n x 32 B.
 * out: n x 32 B.  Returns DALEK_NONE if G or H does not decode (C/ristretto.rs:266-345; `out` is then
 * unspecified), DALEK_E_INVALID_ARG for a scalar with bit 255 set.  The results are those of the
 * reference's Straus; batches of >= 4096 pairs are computed with a fixed-base comb over tables of G
 * and H (same constant-time discipline: masked full-row scans, uniform control flow).  Pinned host
 * buffers let the copies overlap the arithmetic. */
int dalek_b200_ristretto_double_base_batch(dalek_b200_ctx *ctx, const uint8_t *a, const uint8_t *b,
                                           const uint8_t G[32], const uint8_t H[32], size_t n,
                                           uint8_t *out);
/* RistrettoPoint::vartime_multiscalar_mul over compressed Ristretto points
 * (C/ristretto.rs:980-994); result as CompressedRistretto.  Runs like dalek_b200_edwards_vartime_msm, to which the
 * reference forwards (vartime Straus below 190 pairs, host buffers streamed in chunks); DALEK_NONE if a point does
 * not decode (C/ristretto.rs:266-345). */
int dalek_b200_ristretto_vartime_msm(dalek_b200_ctx *ctx, const uint8_t *scalars,
                                     const uint8_t *points, size_t n, uint8_t out_compressed[32]);

/* -------- ed25519 --------------------------------------------------------------------------- */
/*
 * ed25519_dalek::verify_batch (E/batch.rs:146-251).
 *   msgs / msg_lens   n message pointers and lengths          (messages: &[&[u8]])
 *   sigs              n x 64 B R || s                          (signatures: &[Signature])
 *   pubkeys           n x 32 B compressed keys                 (verifying_keys: &[VerifyingKey])
 * In Rust a VerifyingKey already holds its decompressed point (E/verifying.rs:65-71); here keys
 * arrive as bytes and VerifyingKey::from_bytes (E/verifying.rs:167-175) runs inside the call (once
 * per DISTINCT key: repeated keys are de-duplicated on the device): an undecodable key is
 * ED25519_ERR_POINT_DECOMPRESSION.  Then, in the reference's order
 * (E/batch.rs:208-250): non-canonical s -> ED25519_ERR_SCALAR_FORMAT; undecodable R or a
 * non-identity result -> ED25519_ERR_VERIFY; else 0.  No cofactor multiplication.
 * Coefficients z_i: exactly the reference's -- ONE Merlin transcript over the whole batch (batch.rs:168-222), whatever n
 * is.  That transcript is a strictly sequential sponge (1.73 Keccak-f[1600] permutations per signature, one GPU warp:
 * about 11.7 us per signature on an H100, profiles/bench_h100.json), so callers with very large inputs either use ed25519_b200_verify_batches_flat (independent
 * batches, each with the reference's transcript, hashed in parallel) or OPT INTO the option "verify_chunk" = k > 0: one
 * transcript per k consecutive signatures and one combined equation.  The chunked mode is NOT reference-equivalent: its z_i
 * differ from the reference's for n > k, and while the verdict is the same for every batch without small-order components
 * (valid batches pass, invalid ones fail except with probability ~2^-128), for signatures or keys carrying small-order
 * components the un-cofactored equation's verdict depends on the z_i modulo 8 and can differ from the reference's.
 */
int ed25519_b200_verify_batch(dalek_b200_ctx *ctx, const uint8_t *const *msgs, const size_t *msg_lens,
                              const uint8_t *sigs, const uint8_t *pubkeys, size_t n);
/* Same with the messages laid out back to back: message i = msgs_flat[msg_offsets[i] ..
 * msg_offsets[i+1]) (n+1 offsets; the flat-message rule of the hash-to-group block applies to every host-buffer
 * ..._flat call).  Avoids the host-side gather of the pointer form. */
int ed25519_b200_verify_batch_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat,
                                   const uint64_t *msg_offsets, const uint8_t *sigs,
                                   const uint8_t *pubkeys, size_t n);
/* Device-resident variant of the flat form (all four buffers are device pointers). */
int ed25519_b200_verify_batch_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat,
                                       const void *d_msg_offsets, const void *d_sigs,
                                       const void *d_pubkeys, size_t n, size_t msgs_bytes);
/* verify_batch for callers that hold VerifyingKeys: key_points[20 i ..] is the decompressed point of key i (X | Y | Z | T,
 * radix-2^51 limbs, the reference's in-memory EdwardsPoint; what VerifyingKey::from_bytes computed once, E/verifying.rs:
 * 65-71, :167-175) and pubkeys[32 i ..] its encoding (hashed as in batch.rs:179-191).  No key is decompressed inside the
 * call -- the reference's verify_batch does not either (batch.rs:236-238) -- so a batch whose keys are all different costs
 * what a batch with few keys costs.  The points are trusted to be the decodings of the encodings (as a VerifyingKey
 * guarantees); Z = 1 is free, another Z costs one inversion per distinct key.  Never returns POINT_DECOMPRESSION. */
int ed25519_b200_verify_batch_flat_points(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                          const uint8_t *sigs, const uint8_t *pubkeys, const uint64_t *key_points, size_t n);
int ed25519_b200_verify_batch_flat_points_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                              const void *d_sigs, const void *d_pubkeys, const void *d_key_points, size_t n);
/* Many independent batches in one call (SURVEY 8d config 3B: 2^14 batches of 256): signatures
 * [k * batch_size, min(n, (k+1) * batch_size)) form batch k and verdicts[k] receives what
 * ed25519_dalek::verify_batch (batch.rs:146-251) returns for that batch alone (0 / 1 / 3 / 4); each batch
 * uses exactly the reference's transcript (whatever "verify_chunk" is).  A batch passes iff the value E_k of its equation
 * (batch.rs:240-250) is the identity.  The small-order part of every E_k is tested exactly, per batch (it only depends on the
 * scalars modulo 8: S_k = sum (z_i mod 8) R_i + sum ((z_i h_i mod l) mod 8) A_i, [l] S_k == identity) -- sums of batch
 * equations would let the small-order defects of different batches cancel, one input in eight.  For the prime-order parts the
 * combined equation over all undecided batches is tested first (independent transcripts: a non-zero prime-order part
 * leaves it non-zero except with the probability a forgery passes batch.rs itself, ~2^-125); only when it fails are halves
 * re-tested down to single batches, so a clean call costs little more than one large verify_batch, and k failing batches
 * add about k * log2(n / batch_size) partial re-tests.
 * Returns 0 if every verdict is 0, 1 otherwise, negative on engine errors.  verdicts: ceil(n / batch_size) ints (host). */
int ed25519_b200_verify_batches_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat,
                                     const uint64_t *msg_offsets, const uint8_t *sigs,
                                     const uint8_t *pubkeys, size_t n, size_t batch_size, int32_t *verdicts);
int ed25519_b200_verify_batches_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat,
                                         const void *d_msg_offsets, const void *d_sigs,
                                         const void *d_pubkeys, size_t n, size_t batch_size, int32_t *verdicts);
/* The same for callers that hold VerifyingKeys (the reference's bench shape, E/benches/ed25519_benchmarks.rs:56-73: every key
 * different): key_points as in ed25519_b200_verify_batch_flat_points -- no key is decompressed inside the call (batch.rs:236-238). */
int ed25519_b200_verify_batches_flat_points(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                            const uint8_t *sigs, const uint8_t *pubkeys, const uint64_t *key_points, size_t n,
                                            size_t batch_size, int32_t *verdicts);
int ed25519_b200_verify_batches_flat_points_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                                const void *d_sigs, const void *d_pubkeys, const void *d_key_points, size_t n,
                                                size_t batch_size, int32_t *verdicts);
/* Many independent single verifications (SURVEY 8f rank 3): results[i] = what VerifyingKey::from_bytes followed by
 * verify (strict = 0, E/verifying.rs:167-175, :203-219) or verify_strict (strict = 1, E/verifying.rs:359-382)
 * returns for signature i alone: 0 Ok, 1 Verify, 3 ScalarFormat, 4 PointDecompression.  R' = [s]B - [k]A is
 * recomputed (RCompute, E/verifying.rs:496-557) and its ENCODING compared with the signature's R bytes, so --
 * unlike verify_batch -- a non-canonical R is rejected; verify_strict also rejects small-order R or A.
 * When the batch holds few distinct keys (every key signing at least eight signatures on average; option "each_comb") the
 * 64 x 8 multiples (j+1) 16^i A of every distinct key are tabulated once per call and each signature costs 128 mixed
 * additions and no doubling; otherwise every signature pays its own 252 doublings.  Same results either way.
 * Returns 0 if every result is 0, 1 otherwise; negative on engine errors.  results: n bytes (host).  Flat messages as in
 * the hash-to-group block. */
int ed25519_b200_verify_each_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                  const uint8_t *sigs, const uint8_t *pubkeys, size_t n, int strict,
                                  uint8_t *results);
int ed25519_b200_verify_each_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                      const void *d_sigs, const void *d_pubkeys, size_t n, int strict,
                                      uint8_t *results);
/* Debug/parity aid: the 16-byte z_i coefficients drawn in the last verify_batch call. */
int ed25519_b200_last_zs(dalek_b200_ctx *ctx, uint8_t *zs_out, size_t n);

/* -------- ed25519 signing (secret-key operations) ------------------------------------------------
 * Host buffers; each call blocks and streams the batch in pieces like the codecs.  n = 0 is a successful no-op; a NULL
 * buffer with n > 0 is DALEK_E_INVALID_ARG.  Flat messages follow the rule of the hash-to-group block.  Seeds are the
 * 32-byte SecretKeys of SigningKey::from_bytes (E/signing.rs:106).  The signer is constant time in the secrets (the seed,
 * its expansion, the nonce r): uniform control flow, full-row scans of the comb table of B, branch-free arithmetic mod l;
 * only the lengths of the messages and of the context shape the work.  The device copies of the seeds and of their
 * expansions are cleared before a call returns.  No option affects these calls.
 *
 * SigningKey::from_bytes(seed).verifying_key() (E/signing.rs:106, :171; hazmat.rs:84-99): n x 32 B seeds -> n x 32 B
 * VerifyingKey bytes. */
int ed25519_b200_verifying_keys(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n, uint8_t *pubkeys_out);
/* Signer::try_sign -> raw_sign (E/signing.rs:566-571, :854-904): sigs_out n x 64 B, signature i over message i.
 * n_seeds is n (seed i signs message i) or 1 (one key signs every message); any other value is DALEK_E_INVALID_ARG. */
int ed25519_b200_sign_flat(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *msgs_flat,
                           const uint64_t *msg_offsets, size_t n, uint8_t *sigs_out);
/* SigningKey::sign_prehashed -> raw_sign_prehashed (Ed25519ph, E/signing.rs:312, :917-976): prehashes n x 64 B, the
 * finalized MsgDigest of each message (PH(M) = SHA-512(M) for RFC 8032); one context of context_len <= 255 bytes for
 * the batch (NULL only with context_len = 0: None and Some(b"") hash alike).  context_len > 255 returns
 * ED25519_ERR_PREHASHED_CONTEXT_LENGTH.  n_seeds as in sign_flat. */
int ed25519_b200_sign_prehashed(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *prehashes, size_t n,
                                const uint8_t *context, size_t context_len, uint8_t *sigs_out);
/* VerifyingKey::verify_prehashed (strict = 0) / verify_prehashed_strict (strict = 1) (E/verifying.rs:230-257, :424-459)
 * for n independent signatures: results, return value and error precedence as in ed25519_b200_verify_each_flat, with the
 * challenge k = SHA-512(dom2(1, C) || R || A || PH) mod l (RCompute with a prehash context, E/verifying.rs:496-557).
 * prehashes: n x 64 B.  context_len > 255 is DALEK_E_INVALID_ARG (the reference only debug-asserts it). */
int ed25519_b200_verify_prehashed_each(dalek_b200_ctx *ctx, const uint8_t *prehashes, const uint8_t *context,
                                       size_t context_len, const uint8_t *sigs, const uint8_t *pubkeys, size_t n,
                                       int strict, uint8_t *results);

/* -------- resident verifying-key sets -----------------------------------------------------------------------------------
 * A VerifyingKey is decompressed once by VerifyingKey::from_bytes (E/verifying.rs:167-175) and then verifies any number of
 * messages.  A set holds k keys in device memory: the 32 bytes of each key exactly as given (the challenge k = SHA-512(R ||
 * A || M) hashes VerifyingKey.compressed, E/verifying.rs:515-523, so a non-canonical encoding is hashed as the caller
 * wrote it), the 64 x 8 multiples (j+1) 16^i A of each key as FP64 affine Niels (64 KiB per key, the per-key comb tables
 * of ed25519_b200_verify_each_flat), a status byte and a 4-byte slot index per key.  new allocates that memory and
 * destroy frees it; the set is not a context workspace and serves only the context that made it (another context is
 * DALEK_E_INVALID_ARG).
 *
 * new is VerifyingKey::from_bytes once per key, for k >= 1 keys (k = 0 is DALEK_E_INVALID_ARG).  If a key does not
 * decode, ok[i] = 0 for it (ok: k bytes, nullable; 1 for every other key), *out stays NULL, nothing stays allocated and
 * the call returns ED25519_ERR_POINT_DECOMPRESSION.  weak[i] (k bytes, nullable) is VerifyingKey::is_weak
 * (E/verifying.rs:192-194), i.e. EdwardsPoint::is_small_order (C/edwards.rs:1405-1407) of the decoded key, and 0 for a
 * key that does not decode.  A failed allocation returns DALEK_E_NOMEM with last_error set and no set. */
typedef struct ed25519_b200_key_set ed25519_b200_key_set;
int ed25519_b200_key_set_new(dalek_b200_ctx *ctx, const uint8_t *pubkeys /* k x 32 B */, size_t k,
                             uint8_t *ok /* k, nullable */, uint8_t *weak /* k, nullable */, ed25519_b200_key_set **out);
size_t ed25519_b200_key_set_len(const ed25519_b200_key_set *s);
/* destroy waits for the device and frees the set; it does not use the context, so a set may be destroyed before or
 * after its context.  NULL is a no-op. */
void ed25519_b200_key_set_destroy(ed25519_b200_key_set *s);
/* verify (strict = 0, E/verifying.rs:203-219) or verify_strict (strict = 1, E/verifying.rs:359-382) of signature i
 * under key key_idx[i] of the set (key_idx NULL: key 0 for every signature).  results and return value are exactly those
 * of ed25519_b200_verify_each_flat on the same inputs with the key bytes inlined, with the same error precedence: 0 Ok,
 * 1 Verify, 3 ScalarFormat (PointDecompression cannot occur: every key of a set decodes).  verify_strict rejects every
 * signature under a weak key.  The set's tables always serve the call (option "each_comb" does not apply); each signature
 * costs 128 mixed additions and no doubling, with no per-call table build, key de-duplication or host synchronisation.
 * n = 0 is a successful no-op; a NULL sigs or results with n > 0 is DALEK_E_INVALID_ARG; flat messages as in the
 * hash-to-group block.  Host buffers: an index >= k is DALEK_E_INVALID_ARG before any device work, and the batch is
 * streamed in pieces. */
int ed25519_b200_key_set_verify_flat(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint8_t *msgs_flat,
                                     const uint64_t *msg_offsets, const uint8_t *sigs, const uint32_t *key_idx /* n, or NULL */,
                                     size_t n, int strict, uint8_t *results /* n */);
/* same with messages, offsets, signatures and indices in device memory; results in host memory; blocks until done.  An
 * index >= k is never used as an address (key 0 is read in its place) and is reported after the batch ran: the call
 * returns DALEK_E_INVALID_ARG and the results are unspecified. */
int ed25519_b200_key_set_verify_flat_dev(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const void *d_msgs_flat,
                                         const void *d_msg_offsets, const void *d_sigs, const void *d_key_idx, size_t n,
                                         int strict, uint8_t *results /* host */);
/* verify_prehashed (strict = 0) / verify_prehashed_strict (strict = 1) (E/verifying.rs:230-257, :424-459) of signature i
 * under key key_idx[i]: results and return value as ed25519_b200_verify_prehashed_each on the same inputs with the key
 * bytes inlined.  prehashes: n x 64 B; one context of context_len <= 255 bytes (NULL only with context_len = 0), a longer
 * one is DALEK_E_INVALID_ARG.  Other rules as ed25519_b200_key_set_verify_flat. */
int ed25519_b200_key_set_verify_prehashed(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint8_t *prehashes,
                                          const uint8_t *context, size_t context_len, const uint8_t *sigs,
                                          const uint32_t *key_idx /* n, or NULL */, size_t n, int strict, uint8_t *results);

/* -------- hazmat signing from expanded secret keys (secret-key operations) ---------------------------------------------
 * ed25519_dalek::hazmat signs from an ExpandedSecretKey: keys that have no seed, such as hierarchically derived children,
 * blinded keys or scalars from a threshold protocol.  esks holds 64-byte ExpandedSecretKey bytes: the low 32 bytes are
 * the scalar bytes, the high 32 bytes hash_prefix.  ExpandedSecretKey::from_bytes (E/hazmat.rs:84-99) clamps the scalar
 * bytes and reduces them mod l; any 64 bytes are accepted.  Secret: the esks and everything derived from them but the
 * verifying keys and the signatures; constant time in them as the signer above, and their device copies are cleared
 * before a call returns, failed calls included.  Host buffers, streamed in pieces; n = 0 is a successful no-op, a NULL
 * buffer with n > 0 is DALEK_E_INVALID_ARG; flat messages as in the hash-to-group block.  No option affects these calls.
 *
 * VerifyingKey::from(&ExpandedSecretKey::from_bytes(esk)) (E/verifying.rs:97-102): n x 64 B esks -> n x 32 B
 * compress([clamp(lo) mod l]B), which is compress([clamp(lo)]B). */
int ed25519_b200_expanded_verifying_keys(dalek_b200_ctx *ctx, const uint8_t *esks, size_t n, uint8_t *pubkeys_out);
/* hazmat::raw_sign::<Sha512> (E/hazmat.rs:137, E/signing.rs:854-904): sigs_out n x 64 B, signature i over message i under
 * esk i and verifying key i (n_keys = n) or under esks[0] / vks[0] for every message (n_keys = 1; any other value is
 * DALEK_E_INVALID_ARG).  vks (n_keys x 32 B) is hashed into the challenge exactly as given: a key that does not match
 * the secret gives the reference's bytes for that key, not an error.  The call does not decode vks: in the reference the
 * VerifyingKey type guarantees that the bytes decode, here the caller must.  With one key per message this costs one
 * comb per signature, as A is supplied. */
int ed25519_b200_raw_sign_flat(dalek_b200_ctx *ctx, const uint8_t *esks, const uint8_t *vks, size_t n_keys, const uint8_t *msgs_flat,
                               const uint64_t *msg_offsets, size_t n, uint8_t *sigs_out);
/* hazmat::raw_sign_prehashed::<Sha512, Sha512> (Ed25519ph, E/hazmat.rs:182, E/signing.rs:917-976): prehashes n x 64 B,
 * one context for the batch as in ed25519_b200_sign_prehashed (context_len > 255 returns
 * ED25519_ERR_PREHASHED_CONTEXT_LENGTH and writes nothing).  esks, vks and n_keys as in ed25519_b200_raw_sign_flat. */
int ed25519_b200_raw_sign_prehashed(dalek_b200_ctx *ctx, const uint8_t *esks, const uint8_t *vks, size_t n_keys,
                                    const uint8_t *prehashes, size_t n, const uint8_t *context, size_t context_len,
                                    uint8_t *sigs_out);

/* -------- resident signing-key sets (secret-key operations) ------------------------------------------------------------
 * A service that signs at volume holds a fixed set of keys and signs each message under one of them.  A set derives its
 * k keys once and keeps them in device memory: per key the clamped scalar and hash_prefix (64 B, secret) and the
 * verifying key (32 B), plus a host copy of the verifying keys.  new allocates that memory and destroy clears the secret
 * part and frees it; the set is not a context workspace and serves only the context that made it (another context is
 * DALEK_E_INVALID_ARG).  Each signature costs one comb and no key derivation.  Constant time as the signer above; the
 * key indices are public (which key signs a message is not secret in the reference either).
 *
 * new takes k >= 1 keys (k = 0 is DALEK_E_INVALID_ARG) in one form:
 *   DALEK_SIGNING_KEY_SEED      32 B SecretKey each: SigningKey::from_bytes (E/signing.rs:106).
 *   DALEK_SIGNING_KEY_KEYPAIR   64 B seed || public half each: SigningKey::from_keypair_bytes (E/signing.rs:140-150).
 *       status[i] = ED25519_ERR_POINT_DECOMPRESSION when the public half does not decode (checked first, as
 *       VerifyingKey::try_from runs first in the reference), else ED25519_ERR_MISMATCHED_KEYPAIR when it is not
 *       byte-equal to the derived verifying key (equality is on bytes, E/verifying.rs:91-95, so a non-canonical
 *       encoding of the right point is a mismatch).
 *   DALEK_SIGNING_KEY_EXPANDED  64 B ExpandedSecretKey bytes each: ExpandedSecretKey::from_bytes (E/hazmat.rs:84-99),
 *       the verifying key derived as in ed25519_b200_expanded_verifying_keys.
 * Any other form is DALEK_E_INVALID_ARG.  status (k bytes, nullable) is 0 for every key that is fine.  Any nonzero status
 * leaves *out NULL and nothing allocated, and the call returns the status of the first failing key.  A failed allocation
 * returns DALEK_E_NOMEM with last_error set and no set.  The staged secret bytes are cleared before the call returns. */
#define DALEK_SIGNING_KEY_SEED 0
#define DALEK_SIGNING_KEY_KEYPAIR 1
#define DALEK_SIGNING_KEY_EXPANDED 2
typedef struct ed25519_b200_signing_key_set ed25519_b200_signing_key_set;
int ed25519_b200_signing_key_set_new(dalek_b200_ctx *ctx, const uint8_t *keys /* k x 32 or 64 B */, size_t k, int form,
                                     uint8_t *status /* k, nullable */, ed25519_b200_signing_key_set **out);
size_t ed25519_b200_signing_key_set_len(const ed25519_b200_signing_key_set *s);
/* the k x 32 B verifying keys (SigningKey::verifying_key, E/signing.rs:171), from the host copy: no device access.
 * Returns 0, or DALEK_E_INVALID_ARG for a NULL argument. */
int ed25519_b200_signing_key_set_verifying_keys(const ed25519_b200_signing_key_set *s, uint8_t *pubkeys_out);
/* destroy clears the secret device memory, waits for the device and frees the set; it does not use the context, so a
 * set may be destroyed before or after its context.  NULL is a no-op. */
void ed25519_b200_signing_key_set_destroy(ed25519_b200_signing_key_set *s);
/* Signer::try_sign (E/signing.rs:566-571) of message i under key key_idx[i] of the set (key_idx NULL: key 0 for every
 * message): sigs_out n x 64 B, the bytes ed25519_b200_sign_flat gives with that key's seed (or raw_sign with that
 * ExpandedSecretKey and its derived verifying key).  n = 0 is a successful no-op; a NULL sigs_out with n > 0 is
 * DALEK_E_INVALID_ARG; flat messages as in the hash-to-group block.  An index >= k is DALEK_E_INVALID_ARG before any
 * device work.  The batch is streamed in pieces. */
int ed25519_b200_signing_key_set_sign_flat(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const uint8_t *msgs_flat,
                                           const uint64_t *msg_offsets, const uint32_t *key_idx /* n, or NULL */, size_t n,
                                           uint8_t *sigs_out);
/* same with messages, offsets, indices and signatures in device memory; blocks until done.  An index >= k is never used
 * as an address: that message's signature is 64 zero bytes (never a signature under another key, which a caller that
 * ignores the return code could not tell from a good one), every other message is signed, and the call returns
 * DALEK_E_INVALID_ARG after the batch ran. */
int ed25519_b200_signing_key_set_sign_flat_dev(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const void *d_msgs_flat,
                                               const void *d_msg_offsets, const void *d_key_idx, size_t n, void *d_sigs_out);
/* SigningKey::sign_prehashed (Ed25519ph, E/signing.rs:312, :917-976) of prehash i (n x 64 B) under key key_idx[i], one
 * context for the batch as in ed25519_b200_sign_prehashed: context_len > 255 returns ED25519_ERR_PREHASHED_CONTEXT_LENGTH
 * and writes nothing.  Other rules as ed25519_b200_signing_key_set_sign_flat. */
int ed25519_b200_signing_key_set_sign_prehashed(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const uint8_t *prehashes,
                                                const uint8_t *context, size_t context_len, const uint32_t *key_idx /* n, or NULL */,
                                                size_t n, uint8_t *sigs_out);

/* -------- input synthesis (benchmarks / tests): fixed-base multiples and keys + signatures ---- */
/* out[i] = scalars[i] * B as extended limbs (EdwardsPoint::mul_base, C/edwards.rs:918-928).  Public scalars only:
 * variable-time table lookups. */
int dalek_b200_edwards_mul_base_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, size_t n,
                                      uint64_t *out_limbs /* n x 20 */, uint8_t *out_compressed /* n x 32, nullable */);
/* Keys and signatures in one call: seeds n x 32 B -> pubkeys n x 32 B, sigs n x 64 B; ed25519_b200_verifying_keys
 * followed by ed25519_b200_sign_flat with n_seeds = n (constant time); message layout and checks as in verify_batch_flat. */
int ed25519_b200_sign_batch_flat(dalek_b200_ctx *ctx, const uint8_t *seeds, const uint8_t *msgs_flat,
                                 const uint64_t *msg_offsets, size_t n, uint8_t *pubkeys_out,
                                 uint8_t *sigs_out);

#ifdef __cplusplus
}
#endif
#endif
