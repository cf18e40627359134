// point_ops.cu -- batched group operations on Edwards and Ristretto points (point_ops.cuh):
//   Add / Sub, Neg, Group::double, mul_by_cofactor   k_point_op<FMT, ENC>   one thread per item
//   ct_eq / is_identity                              k_point_eq<FMT>        one thread per item
//   Sum over segments                                k_sum_decode<FMT>      one thread per point: decode to FP64 limbs
//                                                    k_sum_chunks           one CTA per chunk: strided runs, a warp
//                                                                           shuffle tree, a shared-memory tree
//                                                    k_sum_finish<ENC>      one thread per segment: encode
// Element-wise calls decode with varmul_load_point, apply the operation on the integer field and encode: Ristretto in the
// thread, Edwards through k_compress_batch (codecs.cu, one inversion per CODEC_K points) from limbs staged in
// WS_POINT_OPS, EXTENDED as canonical limbs.  Host buffers stream through run_pieces; a broadcast operand is staged in
// WS_CALL_SCRATCH.
// The sum cuts every segment into chunks of PS_CHUNK points that never cross a segment boundary (point_ops.cuh, planned
// on the host from the offsets).  Pieces of whole chunks are decoded at one thread per point, at full occupancy whatever
// the segment lengths, then reduced to one partial sum per chunk; segments may span pieces because the partials are
// combined only at the end, by further chunk levels over the partials until every segment has one.
// Constant time in the points: no branch, loop bound or address depends on a coordinate, a decode outcome or an
// equality (decode failures are gathered by a warp reduction and one atomic per warp, whatever the points).  Every call
// clears the engine's copies of its points, intermediates and results before it returns, also after a failed launch.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "pieces.h"
#include "point_load.cuh"
#include "point_ops.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define PO_THREADS 128
#define PO_PIECE ((size_t)1 << 16)     // items per piece of an element-wise call (a multiple of 128 x CODEC_K)
#define PS_CHUNK 1024u                 // points (or partial sums) per chunk of the sum
#define PS_THREADS 128                 // the most threads of a chunk's CTA
#define PS_PIECE (1u << 16)            // the most points per piece of the sum, in whole chunks

// WS_CALL_SCRATCH: the decode-failure word and the two broadcast operands
#define PO_BAD 0
#define PO_BCAST_A 256
#define PO_BCAST_B 512
#define PO_SCRATCH 1024

__device__ __forceinline__ void ps_store(double *__restrict__ o, const ge64_p3 &P)
{
#pragma unroll
    for (int k = 0; k < 5; k++) { o[k] = P.X.v[k]; o[5 + k] = P.Y.v[k]; o[10 + k] = P.Z.v[k]; o[15 + k] = P.T.v[k]; }
}

__device__ __forceinline__ void ps_load(ge64_p3 &P, const double *__restrict__ s)
{
#pragma unroll
    for (int k = 0; k < 5; k++) { P.X.v[k] = s[k]; P.Y.v[k] = s[5 + k]; P.Z.v[k] = s[10 + k]; P.T.v[k] = s[15 + k]; }
}

// item i: op(A_i, B_i) (a_step / b_step 0 broadcast item 0), the identity if an input does not decode; ENC = 1 writes
// CompressedRistretto to enc, ENC = 0 canonical limbs to limbs
template <int FMT, int ENC>
__global__ void __launch_bounds__(PO_THREADS)
k_point_op(const uint32_t *__restrict__ a, size_t a_step, const uint32_t *__restrict__ b, size_t b_step, size_t n, int op,
           uint32_t *__restrict__ enc, uint64_t *__restrict__ limbs, uint8_t *__restrict__ ok, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 A, B, R;
    uint32_t good = varmul_load_point<FMT>(A, a, a_step * i);
    ge_p3_identity(B);
    if (op <= PO_SUB) good &= varmul_load_point<FMT>(B, b, b_step * i);   // the operation is public
    point_apply(R, A, B, op);
    point_cmov_identity(R, 1u - good);
    if (ENC) {
        uint32_t w[8];
        ristretto_compress<1>(w, R);
#pragma unroll
        for (int k = 0; k < 8; k++) enc[8 * i + k] = w[k];
    } else {
        uint64_t l[20];
        point_to_limbs(l, R);
#pragma unroll
        for (int k = 0; k < 20; k++) limbs[20 * i + k] = l[k];
    }
    if (ok) ok[i] = (uint8_t)good;
    warp_report_bad(good, bad);
}

// out[i] = eq | both_decoded << 1; b = NULL compares with the identity
template <int FMT>
__global__ void __launch_bounds__(PO_THREADS)
k_point_eq(const uint32_t *__restrict__ a, size_t a_step, const uint32_t *__restrict__ b, size_t b_step, size_t n, uint32_t rist,
           uint8_t *__restrict__ out, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 A, B;
    uint32_t good = varmul_load_point<FMT>(A, a, a_step * i);
    ge_p3_identity(B);
    if (b) good &= varmul_load_point<FMT>(B, b, b_step * i);          // public: the call compares with the identity
    const uint32_t e = rist ? ristretto_eq(A, B) : edwards_eq(A, B);   // the group is public
    out[i] = (uint8_t)((e & good) | (good << 1));
    warp_report_bad(good, bad);
}

// point i of the piece -> 20 doubles (FP64 limbs at scale 1) and its decode flag; an undecodable point is the identity
template <int FMT>
__global__ void __launch_bounds__(PO_THREADS)
k_sum_decode(const uint32_t *__restrict__ points, size_t n, double *__restrict__ dec, uint8_t *__restrict__ dec_ok)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge_p3 p;
    const uint32_t good = varmul_load_point<FMT>(p, points, i);
    ge64_p3 P;
    ge64_from_p3(P, p);
    ps_store(dec + 20 * i, P);
    dec_ok[i] = (uint8_t)good;
}

// chunk c = c0 + blockIdx.x (items start[c] .. start[c+1], read at index - base) -> partial[c], part_ok[c].  Thread t adds
// items t, t + blockDim.x, ... in order; the lanes of each warp are combined by a shuffle tree, the warps through shared
// memory.  Every bound is the chunk length, which is public.
__global__ void __launch_bounds__(PS_THREADS)
k_sum_chunks(const double *__restrict__ in, const uint8_t *__restrict__ in_ok, uint32_t base, const uint32_t *__restrict__ start,
             uint32_t c0, double *__restrict__ partial, uint8_t *__restrict__ part_ok)
{
    __shared__ double s_warp[PS_THREADS / 32][20];
    const uint32_t c = c0 + blockIdx.x;
    const uint32_t first = start[c] - base, len = start[c + 1] - start[c];
    fe64 d2;
    { fe k; fe_const_2d(k); fe64_from_fe(d2, k); }
    ge64_p3 S, P;
    ge64_identity(S);
    uint32_t good = 1;
#pragma unroll 1
    for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) {
        ps_load(P, in + 20 * (size_t)(first + k));
        good &= in_ok[first + k];
        ge64_add_p3(S, S, P, d2);
    }
    good = (uint32_t)__syncthreads_and((int)good);
    const uint32_t lanes = len < 32 ? len : 32;                        // lanes of a warp that may hold points
#pragma unroll 1
    for (uint32_t d = (1u << (32 - __clz((int)(lanes - 1)))) >> 1; d > 0; d >>= 1) {
        ge64_shfl_down(P, S, (int)d);
        ge64_add_p3(S, S, P, d2);
    }
    const uint32_t nw = min((len + 31) / 32, blockDim.x / 32);   // warps that hold points
    if (nw > 1) {
        const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        if (lane == 0) ps_store(s_warp[wid], S);
        __syncthreads();
        if (wid == 0) {
            if (lane < nw) ps_load(S, s_warp[lane]);
            else ge64_identity(S);
#pragma unroll 1
            for (uint32_t d = (1u << (32 - __clz((int)(nw - 1)))) >> 1; d > 0; d >>= 1) {
                ge64_shfl_down(P, S, (int)d);
                ge64_add_p3(S, S, P, d2);
            }
        }
    }
    if (threadIdx.x == 0) {
        ps_store(partial + 20 * (size_t)c, S);
        part_ok[c] = (uint8_t)good;
    }
}

// segment j: its one partial sum (the identity when it is empty or holds an undecodable point), encoded as
// CompressedRistretto (ENC = 1) or as canonical limbs
template <int ENC>
__global__ void __launch_bounds__(PO_THREADS)
k_sum_finish(const double *__restrict__ partial, const uint8_t *__restrict__ part_ok, const uint32_t *__restrict__ seg_base, size_t m,
             uint32_t *__restrict__ enc, uint64_t *__restrict__ limbs, uint8_t *__restrict__ ok, int *bad)
{
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    ge64_p3 S;
    ge64_identity(S);
    uint32_t good = 1;
    if (seg_base[j + 1] > seg_base[j]) {                               // the segment is not empty (public)
        ps_load(S, partial + 20 * (size_t)seg_base[j]);
        good = part_ok[seg_base[j]];
    }
    ge64_cmov_identity(S, 1u - good);
    ge_p3 q;
    ge64_to_p3(q, S);
    if (ENC) {
        uint32_t w[8];
        ristretto_compress<1>(w, q);
#pragma unroll
        for (int k = 0; k < 8; k++) enc[8 * j + k] = w[k];
    } else {
        uint64_t l[20];
        point_to_limbs(l, q);
#pragma unroll
        for (int k = 0; k < 20; k++) limbs[20 * j + k] = l[k];
    }
    ok[j] = (uint8_t)good;
    warp_report_bad(good, bad);
}

// ---- argument rules ----
// The group of a call (rist) from its input format and flags; out_fmt must be the group's encoding or EXTENDED.
static int po_formats(dalek_b200_ctx *ctx, int in_fmt, int flags, int allowed_flags, int out_fmt, uint32_t &rist)
{
    if (flags & ~allowed_flags) { ctx->last_error = "unknown flag bits"; return DALEK_E_INVALID_ARG; }
    if (in_fmt == DALEK_POINTS_COMPRESSED && !(flags & DALEK_POINT_RISTRETTO)) rist = 0;
    else if (in_fmt == DALEK_POINTS_RISTRETTO) rist = 1;
    else if (in_fmt == DALEK_POINTS_EXTENDED) rist = (flags & DALEK_POINT_RISTRETTO) ? 1u : 0u;
    else { ctx->last_error = "in_fmt must be COMPRESSED, RISTRETTO or EXTENDED, and COMPRESSED is Edwards"; return DALEK_E_INVALID_ARG; }
    if (out_fmt != DALEK_POINTS_EXTENDED && out_fmt != (rist ? DALEK_POINTS_RISTRETTO : DALEK_POINTS_COMPRESSED)) {
        ctx->last_error = "out_fmt must be the group's own encoding or EXTENDED";
        return DALEK_E_INVALID_ARG;
    }
    return 0;
}

static size_t po_out_bytes(int out_fmt) { return out_fmt == DALEK_POINTS_EXTENDED ? 160 : 32; }

// ---- element-wise calls ----
// what one call runs: input format, output format (0 for equality), operation, group and its device scratch
struct PoCall {
    int fmt, out_fmt, op;
    bool eq;
    uint32_t rist;
    int *bad;
    uint64_t *slot[2];      // Edwards results as limbs before their encoding, one slot per stream
};

// one piece of m items on stream st (k: the piece's index); returns the number of kernels it enqueued
template <int FMT>
static int po_launch_fmt(const PoCall &c, const void *a, size_t as, const void *b, size_t bs, size_t m, void *out, uint8_t *ok, size_t k,
                         cudaStream_t st)
{
    const unsigned g = cdiv(m, PO_THREADS);
    const uint32_t *pa = (const uint32_t *)a, *pb = (const uint32_t *)b;
    if (c.eq) {
        k_point_eq<FMT><<<g, PO_THREADS, 0, st>>>(pa, as, pb, bs, m, c.rist, (uint8_t *)out, c.bad);
        return 1;
    }
    if constexpr (FMT != DALEK_POINTS_COMPRESSED) {
        if (c.out_fmt == DALEK_POINTS_RISTRETTO) {
            k_point_op<FMT, 1><<<g, PO_THREADS, 0, st>>>(pa, as, pb, bs, m, c.op, (uint32_t *)out, nullptr, ok, c.bad);
            return 1;
        }
    }
    if (c.out_fmt == DALEK_POINTS_EXTENDED) {
        k_point_op<FMT, 0><<<g, PO_THREADS, 0, st>>>(pa, as, pb, bs, m, c.op, nullptr, (uint64_t *)out, ok, c.bad);
        return 1;
    }
    uint64_t *l = c.slot[k & 1];
    k_point_op<FMT, 0><<<g, PO_THREADS, 0, st>>>(pa, as, pb, bs, m, c.op, nullptr, l, ok, c.bad);
    edwards_compress_enqueue(l, m, (uint32_t *)out, st);
    return 2;
}

static int po_launch(const PoCall &c, const void *a, size_t as, const void *b, size_t bs, size_t m, void *out, uint8_t *ok, size_t k,
                     cudaStream_t st)
{
    if (c.fmt == DALEK_POINTS_EXTENDED) return po_launch_fmt<DALEK_POINTS_EXTENDED>(c, a, as, b, bs, m, out, ok, k, st);
    if (c.fmt == DALEK_POINTS_RISTRETTO) return po_launch_fmt<DALEK_POINTS_RISTRETTO>(c, a, as, b, bs, m, out, ok, k, st);
    return po_launch_fmt<DALEK_POINTS_COMPRESSED>(c, a, as, b, bs, m, out, ok, k, st);
}

// clear what the call left on the device (inputs, intermediates, results), up to what each workspace holds, then wait;
// the call's result is its first failure, else the wipe's
static int po_finish(dalek_b200_ctx *ctx, int rc, size_t in_bytes, size_t out_bytes, size_t ops_bytes)
{
    auto clear = [&](DevBuf &w, size_t bytes) {
        if (w.p && bytes && cudaMemsetAsync(w.p, 0, std::min(bytes, w.cap), ctx->stream) != cudaSuccess) return false;
        return true;
    };
    bool good = clear(ctx->ws[WS_STAGING_IN], in_bytes) && clear(ctx->ws[WS_STAGING_OUT], out_bytes) &&
                clear(ctx->ws[WS_CALL_SCRATCH], PO_SCRATCH) && clear(ctx->ws[WS_POINT_OPS], ops_bytes);
    good = cudaStreamSynchronize(ctx->stream) == cudaSuccess && good;
    if (!good && !rc) { ctx->last_error = "clearing the call's device buffers failed"; rc = DALEK_E_CUDA; }
    return rc;
}

// the decode-failure word, read back after the stream's work
static int po_read_bad(dalek_b200_ctx *ctx, const int *d_bad, int *bad)
{
    int rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *bad = *(const int *)ctx->h_pinned;
    return 0;
}

// Every element-wise call after its argument checks: n items of op(A_i, B_i) (eq: the comparison), a and b with steps
// n_a, n_b in {1, n} (b may be NULL for unary operations and for the identity).
static int po_run(dalek_b200_ctx *ctx, PoCall c, const void *a, size_t n_a, const void *b, size_t n_b, size_t n, void *out, uint8_t *ok,
                  bool on_device)
{
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const size_t pin = msm_point_bytes(c.fmt), out_sz = c.eq ? 1 : po_out_bytes(c.out_fmt);
    const bool ba = n_a == 1, bb = b && n_b == 1;
    const size_t slot_bytes = c.eq || c.out_fmt != DALEK_POINTS_COMPRESSED ? 0 : std::min(n, PO_PIECE) * 160;
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], PO_SCRATCH))) return rc;
    if (slot_bytes && (rc = ws_reserve(ctx, ctx->ws[WS_POINT_OPS], 2 * slot_bytes))) return rc;
    char *scratch = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    c.bad = (int *)(scratch + PO_BAD);
    c.slot[0] = (uint64_t *)ctx->ws[WS_POINT_OPS].p;
    c.slot[1] = (uint64_t *)((char *)ctx->ws[WS_POINT_OPS].p + slot_bytes);
    const size_t a_sz = ba ? 0 : pin, b_sz = (!b || bb) ? 0 : pin, ok_sz = ok ? 1 : 0;
    rc = 0;
    if (cudaMemsetAsync(c.bad, 0, 4, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
    if (!rc && !on_device) {
        if (ba && cudaMemcpyAsync(scratch + PO_BCAST_A, a, pin, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        if (bb && cudaMemcpyAsync(scratch + PO_BCAST_B, b, pin, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
    }
    if (!rc && !on_device) {
        const void *bcast_b = b ? (const void *)(scratch + PO_BCAST_B) : nullptr;
        rc = run_pieces(ctx, nullptr, nullptr, ba ? nullptr : (const uint8_t *)a, a_sz, b_sz ? (const uint8_t *)b : nullptr, b_sz,
                        (uint8_t *)out, out_sz, ok, ok_sz, n,
                        [&](const uint8_t *, const uint64_t *, const uint8_t *d_a, const uint8_t *d_b, size_t m, uint8_t *d_o,
                            uint8_t *d_ok, cudaStream_t st, size_t lo) {
                            const void *pa = ba ? (const void *)(scratch + PO_BCAST_A) : (const void *)d_a;
                            const void *pb = bb ? bcast_b : (b ? (const void *)d_b : nullptr);
                            ctx->launches += po_launch(c, pa, ba ? 0 : 1, pb, bb ? 0 : 1, m, d_o, ok ? d_ok : nullptr, lo / PO_PIECE, st) - 1;
                            return 0;
                        },
                        PO_PIECE);
    } else if (!rc) {
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
        size_t k = 0;
        for (size_t lo = 0; lo < n; lo += PO_PIECE, k++) {
            const size_t m = std::min(PO_PIECE, n - lo);
            const void *pa = (const char *)a + (ba ? 0 : lo * pin);
            const void *pb = b ? (const void *)((const char *)b + (bb ? 0 : lo * pin)) : nullptr;
            ctx->launches += po_launch(c, pa, ba ? 0 : 1, pb, bb ? 0 : 1, m, (char *)out + lo * out_sz, ok ? ok + lo : nullptr, k,
                                       ctx->stream);
            if (cudaGetLastError() != cudaSuccess) { ctx->last_error = "kernel launch failed"; rc = DALEK_E_CUDA; break; }
        }
        if (!rc && cudaEventRecord(ctx->ev_b, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        ctx->last_kernel_launches = (int)k;
    }
    int bad = 0;
    if (!rc) rc = po_read_bad(ctx, c.bad, &bad);
    if (on_device && !rc) {
        float ms = 0.f;
        if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    }
    rc = po_finish(ctx, rc, on_device ? 0 : n * (a_sz + b_sz), on_device ? 0 : n * (out_sz + ok_sz), 2 * slot_bytes);
    if (rc) return rc;
    return bad ? DALEK_NONE : DALEK_OK;
}

static int po_add(dalek_b200_ctx *ctx, const void *a, size_t n_a, const void *b, size_t n_b, int in_fmt, size_t n, int flags, int out_fmt,
                  void *out, uint8_t *ok, bool on_device)
{
    if (!ctx || (n && (!a || !b || !out))) return DALEK_E_INVALID_ARG;
    if ((n_a != 1 && n_a != n) || (n_b != 1 && n_b != n)) { ctx->last_error = "n_a and n_b must each be 1 or n"; return DALEK_E_INVALID_ARG; }
    PoCall c{};
    int rc;
    if ((rc = po_formats(ctx, in_fmt, flags, DALEK_POINT_SUB | DALEK_POINT_RISTRETTO, out_fmt, c.rist))) return rc;
    c.fmt = in_fmt; c.out_fmt = out_fmt; c.op = (flags & DALEK_POINT_SUB) ? PO_SUB : PO_ADD;
    return po_run(ctx, c, a, n_a, b, n_b, n, out, ok, on_device);
}

static int po_unary(dalek_b200_ctx *ctx, int op, const void *points, int in_fmt, size_t n, int flags, int out_fmt, void *out, uint8_t *ok,
                    bool on_device)
{
    if (!ctx || (n && (!points || !out))) return DALEK_E_INVALID_ARG;
    PoCall c{};
    int rc;
    if ((rc = po_formats(ctx, in_fmt, flags, DALEK_POINT_RISTRETTO, out_fmt, c.rist))) return rc;
    if (op != DALEK_POINT_NEG && op != DALEK_POINT_DOUBLE && op != DALEK_POINT_MUL_BY_COFACTOR) {
        ctx->last_error = "op must be DALEK_POINT_NEG, DALEK_POINT_DOUBLE or DALEK_POINT_MUL_BY_COFACTOR";
        return DALEK_E_INVALID_ARG;
    }
    if (op == DALEK_POINT_MUL_BY_COFACTOR && c.rist) {
        ctx->last_error = "mul_by_cofactor is defined for Edwards points only";
        return DALEK_E_INVALID_ARG;
    }
    c.fmt = in_fmt; c.out_fmt = out_fmt;
    c.op = op == DALEK_POINT_NEG ? PO_NEG : op == DALEK_POINT_DOUBLE ? PO_DOUBLE : PO_COFACTOR;
    return po_run(ctx, c, points, n, nullptr, 0, n, out, ok, on_device);
}

// ---- the segmented sum ----
// the device arrays of one call, carved from WS_POINT_OPS
struct PsSlot {
    double *dec[2]; uint8_t *dec_ok[2];     // decoded points of the pieces on each stream
    std::vector<uint32_t *> start;          // per level: the chunks' first items
    uint32_t *seg_base;                     // the last level's chunk of each segment
    double *part[2]; uint8_t *part_ok[2];   // partial sums of the even and odd levels
    uint64_t *limbs; uint32_t *enc; uint8_t *ok;
    size_t bytes;
};

static void ps_carve(PsSlot &s, char *p, const std::vector<PsLevel> &lv, size_t m, size_t piece_pts)
{
    size_t at = 0;
    auto take = [&](size_t b) { char *q = p ? p + at : nullptr; at += (b + 255) & ~(size_t)255; return q; };
    for (int k = 0; k < 2; k++) { s.dec[k] = (double *)take(piece_pts * 160); s.dec_ok[k] = (uint8_t *)take(piece_pts); }
    s.start.resize(lv.size());
    for (size_t l = 0; l < lv.size(); l++) s.start[l] = (uint32_t *)take(lv[l].start.size() * 4);
    s.seg_base = (uint32_t *)take((m + 1) * 4);
    for (int k = 0; k < 2; k++) {
        const size_t np = lv.size() > (size_t)k ? lv[k].start.size() - 1 : 0;   // levels k, k + 2, ... are no larger
        s.part[k] = (double *)take(np * 160);
        s.part_ok[k] = (uint8_t *)take(np);
    }
    s.limbs = (uint64_t *)take(m * 160);
    s.enc = (uint32_t *)take(m * 32);
    s.ok = (uint8_t *)take(m);
    s.bytes = at;
}

// threads of a chunk's CTA: enough warps for the longest chunk, at most PS_THREADS
static unsigned ps_threads(uint32_t max_len)
{
    return (unsigned)std::min<uint32_t>(PS_THREADS, std::max<uint32_t>(32, (max_len + 31) / 32 * 32));
}

template <int FMT>
static void ps_decode_fmt(const void *pts, size_t n, double *dec, uint8_t *dec_ok, cudaStream_t st)
{
    k_sum_decode<FMT><<<cdiv(n, PO_THREADS), PO_THREADS, 0, st>>>((const uint32_t *)pts, n, dec, dec_ok);
}

static int ps_run(dalek_b200_ctx *ctx, const void *points, int in_fmt, int flags, const uint64_t *offsets, size_t m, int out_fmt, void *out,
                  uint8_t *ok, bool on_device)
{
    if (!ctx || (m && (!offsets || !out))) return DALEK_E_INVALID_ARG;
    uint32_t rist;
    int rc;
    if ((rc = po_formats(ctx, in_fmt, flags, DALEK_POINT_RISTRETTO, out_fmt, rist))) return rc;
    if (!m) return DALEK_OK;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const uint64_t *h_off = offsets;
    std::vector<uint64_t> off_copy;
    if (on_device) {                       // the sizes decide the chunks and the grids: 8 bytes per segment come back
        off_copy.resize(m + 1);
        CUDA_TRY(ctx, cudaMemcpyAsync(off_copy.data(), offsets, (m + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        h_off = off_copy.data();
    }
    if (!ps_offsets_ok(h_off, m)) { ctx->last_error = "offsets must start at 0, not decrease and end below 2^31"; return DALEK_E_INVALID_ARG; }
    const size_t total = (size_t)h_off[m], pin = msm_point_bytes(in_fmt), out_sz = po_out_bytes(out_fmt);
    if (total && !points) return DALEK_E_INVALID_ARG;
    CallTimer timer(ctx);
    std::vector<PsLevel> lv(1);
    ps_plan_level(lv[0], h_off, m, PS_CHUNK);
    while (lv.back().max_per_seg > 1) {
        PsLevel next;
        ps_plan_level(next, lv.back().base.data(), m, PS_CHUNK);
        lv.push_back(std::move(next));
    }
    std::vector<uint32_t> cuts;
    ps_pieces(cuts, lv[0].start, PS_PIECE);
    PsSlot s;
    const size_t piece_pts = std::min<size_t>(total, PS_PIECE);
    ps_carve(s, nullptr, lv, m, piece_pts);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_POINT_OPS], s.bytes))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], PO_SCRATCH))) return rc;
    if (!on_device && (rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, total) * pin))) return rc;
    ps_carve(s, (char *)ctx->ws[WS_POINT_OPS].p, lv, m, piece_pts);
    int *d_bad = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + PO_BAD);
    const uint8_t *staged = (const uint8_t *)ctx->ws[WS_STAGING_IN].p;
    // results: straight into the caller's device buffers, or into the workspace and back to the host
    uint32_t *d_enc = on_device && out_fmt != DALEK_POINTS_EXTENDED ? (uint32_t *)out : s.enc;
    uint64_t *d_limbs = on_device && out_fmt == DALEK_POINTS_EXTENDED ? (uint64_t *)out : s.limbs;
    uint8_t *d_ok = on_device && ok ? ok : s.ok;
    auto body = [&]() -> int {
        CUDA_TRY(ctx, cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
        for (size_t l = 0; l < lv.size(); l++)
            CUDA_TRY(ctx, cudaMemcpyAsync(s.start[l], lv[l].start.data(), lv[l].start.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(s.seg_base, lv.back().base.data(), (m + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
        cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
        const unsigned thr0 = ps_threads(lv[0].max_len);
        for (size_t k = 0; k + 1 < cuts.size(); k++) {       // level 0: pieces of whole chunks over the two streams
            const uint32_t c0 = cuts[k], c1 = cuts[k + 1], p0 = lv[0].start[c0], p1 = lv[0].start[c1];
            cudaStream_t st = ss[k & 1];
            const uint8_t *src;
            if (on_device) src = (const uint8_t *)points + (size_t)p0 * pin;
            else {
                CUDA_TRY(ctx, cudaMemcpyAsync((void *)(staged + (size_t)p0 * pin), (const uint8_t *)points + (size_t)p0 * pin,
                                              (size_t)(p1 - p0) * pin, cudaMemcpyHostToDevice, st));
                src = staged + (size_t)p0 * pin;
            }
            if (in_fmt == DALEK_POINTS_EXTENDED) ps_decode_fmt<DALEK_POINTS_EXTENDED>(src, p1 - p0, s.dec[k & 1], s.dec_ok[k & 1], st);
            else if (in_fmt == DALEK_POINTS_RISTRETTO) ps_decode_fmt<DALEK_POINTS_RISTRETTO>(src, p1 - p0, s.dec[k & 1], s.dec_ok[k & 1], st);
            else ps_decode_fmt<DALEK_POINTS_COMPRESSED>(src, p1 - p0, s.dec[k & 1], s.dec_ok[k & 1], st);
            k_sum_chunks<<<c1 - c0, thr0, 0, st>>>(s.dec[k & 1], s.dec_ok[k & 1], p0, s.start[0], c0, s.part[0], s.part_ok[0]);
            ctx->launches += 2;
            CUDA_TRY(ctx, cudaGetLastError());
        }
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
        for (size_t l = 1; l < lv.size(); l++) {              // the partial sums, until every segment has one
            const uint32_t nch = (uint32_t)lv[l].start.size() - 1;
            k_sum_chunks<<<nch, ps_threads(lv[l].max_len), 0, ctx->stream>>>(s.part[(l - 1) & 1], s.part_ok[(l - 1) & 1], 0, s.start[l], 0,
                                                                              s.part[l & 1], s.part_ok[l & 1]);
            ctx->launches++;
            CUDA_TRY(ctx, cudaGetLastError());
        }
        const size_t L = lv.size() - 1;
        if (out_fmt == DALEK_POINTS_RISTRETTO)
            k_sum_finish<1><<<cdiv(m, PO_THREADS), PO_THREADS, 0, ctx->stream>>>(s.part[L & 1], s.part_ok[L & 1], s.seg_base, m, d_enc,
                                                                                 nullptr, d_ok, d_bad);
        else
            k_sum_finish<0><<<cdiv(m, PO_THREADS), PO_THREADS, 0, ctx->stream>>>(s.part[L & 1], s.part_ok[L & 1], s.seg_base, m, nullptr,
                                                                                 d_limbs, d_ok, d_bad);
        ctx->launches++;
        if (out_fmt == DALEK_POINTS_COMPRESSED) { edwards_compress_enqueue(d_limbs, m, d_enc, ctx->stream); ctx->launches++; }
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
        if (!on_device) {
            const void *src = out_fmt == DALEK_POINTS_EXTENDED ? (const void *)d_limbs : (const void *)d_enc;
            CUDA_TRY(ctx, cudaMemcpyAsync(out, src, m * out_sz, cudaMemcpyDeviceToHost, ctx->stream));
            if (ok) CUDA_TRY(ctx, cudaMemcpyAsync(ok, d_ok, m, cudaMemcpyDeviceToHost, ctx->stream));
        }
        return 0;
    };
    rc = body();
    int bad = 0;
    if (!rc) rc = po_read_bad(ctx, d_bad, &bad);
    if (!rc) {
        float ms = 0.f;
        if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
        ctx->last_kernel_launches = (int)(cuts.size() - 1);
    }
    rc = po_finish(ctx, rc, on_device ? 0 : total * pin, 0, s.bytes);
    if (rc) return rc;
    return bad ? DALEK_NONE : DALEK_OK;
}

extern "C" {

int dalek_b200_point_add_batch(dalek_b200_ctx *ctx, const void *a, size_t n_a, const void *b, size_t n_b, int in_fmt, size_t n, int flags,
                               int out_fmt, void *out, uint8_t *ok)
{
    return po_add(ctx, a, n_a, b, n_b, in_fmt, n, flags, out_fmt, out, ok, false);
}

int dalek_b200_point_add_batch_dev(dalek_b200_ctx *ctx, const void *d_a, size_t n_a, const void *d_b, size_t n_b, int in_fmt, size_t n,
                                   int flags, int out_fmt, void *d_out, void *d_ok)
{
    return po_add(ctx, d_a, n_a, d_b, n_b, in_fmt, n, flags, out_fmt, d_out, (uint8_t *)d_ok, true);
}

int dalek_b200_point_unary_batch(dalek_b200_ctx *ctx, int op, const void *points, int in_fmt, size_t n, int flags, int out_fmt, void *out,
                                 uint8_t *ok)
{
    return po_unary(ctx, op, points, in_fmt, n, flags, out_fmt, out, ok, false);
}

int dalek_b200_point_unary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_points, int in_fmt, size_t n, int flags, int out_fmt,
                                     void *d_out, void *d_ok)
{
    return po_unary(ctx, op, d_points, in_fmt, n, flags, out_fmt, d_out, (uint8_t *)d_ok, true);
}

int dalek_b200_point_eq_batch(dalek_b200_ctx *ctx, const void *a, size_t n_a, const void *b, size_t n_b, int in_fmt, size_t n, int flags,
                              uint8_t *out)
{
    if (!ctx || (n && (!a || !out))) return DALEK_E_INVALID_ARG;
    if ((n_a != 1 && n_a != n) || (b && n_b != 1 && n_b != n)) { ctx->last_error = "n_a and n_b must each be 1 or n"; return DALEK_E_INVALID_ARG; }
    PoCall c{};
    int rc;
    if ((rc = po_formats(ctx, in_fmt, flags, DALEK_POINT_RISTRETTO, DALEK_POINTS_EXTENDED, c.rist))) return rc;
    c.fmt = in_fmt; c.out_fmt = 0; c.eq = true;
    return po_run(ctx, c, a, n_a, b, n_b, n, out, nullptr, false);
}

int dalek_b200_point_sum_batch(dalek_b200_ctx *ctx, const void *points, int in_fmt, int flags, const uint64_t *offsets, size_t m, int out_fmt,
                               void *out, uint8_t *ok)
{
    return ps_run(ctx, points, in_fmt, flags, offsets, m, out_fmt, out, ok, false);
}

int dalek_b200_point_sum_batch_dev(dalek_b200_ctx *ctx, const void *d_points, int in_fmt, int flags, const void *d_offsets, size_t m,
                                   int out_fmt, void *d_out, void *d_ok)
{
    return ps_run(ctx, d_points, in_fmt, flags, (const uint64_t *)d_offsets, m, out_fmt, d_out, (uint8_t *)d_ok, true);
}

}  // extern "C"
