// msm_batch.cu -- m independent multiscalar multiplications in one call: MSM j is the sum of s_i P_i over its own
// segment [offsets[j], offsets[j+1]) of the flat scalar and point arrays, with one result per MSM.
//   VartimeMultiscalarMul::optional_multiscalar_mul   C/traits.rs:196-262, edwards.rs:1002-1030, ristretto.rs:979-994
//   MultiscalarMul::multiscalar_mul                   C/traits.rs:78-134, edwards.rs:970-995, ristretto.rs:964-977
//
// The single-MSM paths give every term its own accumulator and its own 256 doublings, which is right for the latency
// of one small MSM and wasteful for many.  Here the terms of an MSM share an accumulator as in the reference
// (straus.rs:129-138, :181-197): every MSM is cut into chunks of MB_CHUNK terms (msm_batch.cuh) and
//   k_mb_prepare   one thread per term: decode the point, its digits and its table of eight projective Niels points
//   k_mb_chunks    one thread per chunk: the chunk loop of the mode on the FP64 field; one partial sum per chunk
//   k_mb_finish    one thread per MSM: the sum of its partial sums, encoded in the convention of its point format
// The batch runs in pieces of whole MSMs of at most MB_PIECE_TERMS terms, alternating over the context's two streams
// with a workspace each, so the workspace is bounded and the copies of host buffers hide under arithmetic.  A variable-
// time MSM of MB_LARGE_MIN terms or more runs through the single-MSM bucket pipeline inside the same call.
//
// Constant-time mode: no branch, loop bound or address depends on a scalar (msm_batch.cuh); segment sizes and points
// are public.  The one exception is the report of a scalar with bit 255 set by a device-buffer call, which fails the
// call.  Constant-time calls clear the engine's copies of the scalars, digits, tables and partial sums before they return.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "msm_batch.cuh"
#include "point_load.cuh"

#define MB_THREADS 128
#define MB_PIECE_TERMS ((size_t)1 << 18)   // terms per piece: 256 MiB of tables in each of the two workspaces
#define MB_PIECE_SEGS ((size_t)1 << 18)    // MSMs per piece (bounds the result staging when most MSMs are empty)
#define MB_LARGE_MIN ((size_t)1 << 15)     // variable-time MSMs from this size use the bucket pipeline (DESIGN.md §6)

enum { MB_BAD_POINT = 1, MB_BAD_SCALAR = 2 };

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

// Term i of the piece (absolute index t0 + i): its digits and its table.  An undecodable point counts as the identity
// and clears the flag of the MSM that owns it.
template <int FMT, bool CT>
__global__ void __launch_bounds__(MB_THREADS)
k_mb_prepare(const uint32_t *__restrict__ scalars, const uint32_t *__restrict__ points, size_t n, const uint64_t *__restrict__ offsets,
             uint32_t nseg, uint64_t t0, int8_t *__restrict__ digits, ge_pniels_packed *__restrict__ tables, uint8_t *__restrict__ ok,
             int *status)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = scalars[8 * i + k];
    ge_p3 p;
    const uint32_t good = varmul_load_point<FMT>(p, points, i);
    if (!good) {                                                   // the point is public
        uint32_t lo = 0, hi = nseg;                                // offsets[lo] <= t0 + i < offsets[hi]
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (offsets[mid] <= t0 + i) lo = mid; else hi = mid;
        }
        ok[lo] = 0;
        atomicOr(status, MB_BAD_POINT);
    }
    ge64_p3 P;
    ge64_from_p3(P, p);
    ge_pniels_packed tab[8];
    if (CT) {
        if (s[7] >> 31) atomicOr(status, MB_BAD_SCALAR);           // Scalar invariant #1: the call fails
        int8_t d[64];
        mb_radix16(d, s);
        uint32_t *o = reinterpret_cast<uint32_t *>(digits + 64 * i);
#pragma unroll
        for (int k = 0; k < 16; k++)
            o[k] = (uint32_t)(uint8_t)d[4 * k] | ((uint32_t)(uint8_t)d[4 * k + 1] << 8) | ((uint32_t)(uint8_t)d[4 * k + 2] << 16) |
                   ((uint32_t)(uint8_t)d[4 * k + 3] << 24);
        mb_table8(tab, P);
    } else {
        naf5(digits + NAF_LEN * i, s);
        straus_table5(tab, P);
    }
#pragma unroll 1
    for (int e = 0; e < 8; e++) {
        uint4 *o = reinterpret_cast<uint4 *>(tables + 8 * i + e);
#pragma unroll
        for (int k = 0; k < 8; k++) o[k] = make_uint4(tab[e].w[4 * k], tab[e].w[4 * k + 1], tab[e].w[4 * k + 2], tab[e].w[4 * k + 3]);
    }
}

// Chunk c of the piece -> partial[c] (20 doubles: X | Y | Z | T at scale 1)
template <bool CT>
__global__ void __launch_bounds__(MB_THREADS)
k_mb_chunks(const int8_t *__restrict__ digits, const ge_pniels_packed *__restrict__ tables, const uint64_t *__restrict__ offsets,
            const uint32_t *__restrict__ chunk_base, uint32_t nseg, uint32_t nchunks, uint64_t t0, double *__restrict__ partial)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    uint32_t seg, len;
    uint64_t first;
    mb_task(seg, first, len, offsets, chunk_base, nseg, c);
    const size_t i = (size_t)(first - t0);
    ge64_p3 Q;
    if (CT) mb_chunk_ct(Q, digits + 64 * i, tables + 8 * i, len);
    else mb_chunk_vt(Q, digits + NAF_LEN * i, tables + 8 * i, len);
    double *o = partial + 20 * (size_t)c;
#pragma unroll
    for (int k = 0; k < 5; k++) { o[k] = Q.X.v[k]; o[5 + k] = Q.Y.v[k]; o[10 + k] = Q.Z.v[k]; o[15 + k] = Q.T.v[k]; }
}

// MSM j of the piece: the sum of its chunks (the identity for an empty MSM or one with an undecodable point),
// encoded as CompressedEdwardsY or, for Ristretto points, CompressedRistretto; canonical limbs on request
template <int FMT>
__global__ void __launch_bounds__(MB_THREADS)
k_mb_finish(const double *__restrict__ partial, const uint32_t *__restrict__ chunk_base, uint32_t nseg, const uint8_t *__restrict__ ok,
            uint32_t *__restrict__ out, uint64_t *__restrict__ limbs)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nseg) return;
    fe64 d2; fe64_const_2d(d2);
    ge64_p3 Q;
    ge64_identity(Q);
    const uint32_t c1 = ok[j] ? chunk_base[j + 1] : chunk_base[j];
#pragma unroll 1
    for (uint32_t c = chunk_base[j]; c < c1; c++) {
        const double *s = partial + 20 * (size_t)c;
        ge64_p3 R;
#pragma unroll
        for (int k = 0; k < 5; k++) { R.X.v[k] = s[k]; R.Y.v[k] = s[5 + k]; R.Z.v[k] = s[10 + k]; R.T.v[k] = s[15 + k]; }
        ge64_add_p3(Q, Q, R, d2);
    }
    ge_p3 q;
    ge64_to_p3(q, Q);
    uint32_t w[8];
    if (FMT == DALEK_POINTS_RISTRETTO) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * (size_t)j + k] = w[k];
    if (limbs) {
        uint64_t *l = limbs + 20 * (size_t)j;
        fe_to_limbs51(l, q.X); fe_to_limbs51(l + 5, q.Y); fe_to_limbs51(l + 10, q.Z); fe_to_limbs51(l + 15, q.T);
    }
}

// one piece: MSMs [j0, j1) with terms [t0, t1) in nchunks chunks; chunk_base indexes the plan's array
struct MbPiece { size_t j0, j1; uint64_t t0, t1; uint32_t nchunks; size_t cb; };

struct MbPlan {
    std::vector<MbPiece> pieces;
    std::vector<size_t> large;             // MSMs that run through the single-MSM pipeline
    std::vector<uint32_t> chunk_base;      // per piece: j1 - j0 + 1 slots
    size_t max_terms = 0, max_segs = 0, max_chunks = 0;
};

// The batch as runs of whole MSMs: a piece closes before the MSM that would take it past MB_PIECE_TERMS terms or
// MB_PIECE_SEGS MSMs (an MSM larger than a piece is a piece of its own), and around a large variable-time MSM.
static void mb_plan(MbPlan &pl, const uint64_t *offsets, size_t m, bool ct)
{
    size_t j0 = 0;
    auto close = [&](size_t j1) {
        if (j1 == j0) return;
        MbPiece p{j0, j1, offsets[j0], offsets[j1], 0, pl.chunk_base.size()};
        for (size_t j = j0; j < j1; j++) { pl.chunk_base.push_back(p.nchunks); p.nchunks += mb_chunks(offsets[j + 1] - offsets[j]); }
        pl.chunk_base.push_back(p.nchunks);
        pl.max_terms = std::max<size_t>(pl.max_terms, p.t1 - p.t0);
        pl.max_segs = std::max(pl.max_segs, j1 - j0);
        pl.max_chunks = std::max<size_t>(pl.max_chunks, p.nchunks);
        pl.pieces.push_back(p);
        j0 = j1;
    };
    for (size_t j = 0; j < m; j++) {
        const uint64_t nj = offsets[j + 1] - offsets[j];
        if (!ct && nj >= MB_LARGE_MIN) { close(j); pl.large.push_back(j); j0 = j + 1; continue; }
        if (j > j0 && (offsets[j + 1] - offsets[j0] > MB_PIECE_TERMS || j - j0 >= MB_PIECE_SEGS)) close(j);
    }
    close(m);
}

static bool mb_offsets_ok(const uint64_t *offsets, size_t m)
{
    if (offsets[0] != 0) return false;
    for (size_t j = 0; j < m; j++)
        if (offsets[j] > offsets[j + 1]) return false;
    return offsets[m] < (1ull << 31);
}

// the device arrays of one piece, carved from one workspace
struct MbSlot {
    int *status;
    uint64_t *offsets; uint32_t *chunk_base; uint8_t *ok; uint32_t *out; uint64_t *limbs;
    uint32_t *scalars, *points; int8_t *digits; ge_pniels_packed *tables; double *partial;
    size_t secret0, bytes;                  // [secret0, bytes): scalars, points, digits, tables and partial sums
};

static void mb_carve(MbSlot &s, char *base, size_t terms, size_t segs, size_t chunks, size_t pin, bool ct, bool staged)
{
    size_t at = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + at : nullptr; at += (bytes + 255) & ~(size_t)255; return p; };
    s.status = (int *)take(4);
    s.offsets = (uint64_t *)take((segs + 1) * 8);
    s.chunk_base = (uint32_t *)take((segs + 1) * 4);
    s.ok = (uint8_t *)take(segs);
    s.out = (uint32_t *)take(segs * 32);
    s.limbs = (uint64_t *)take(segs * 160);
    s.secret0 = at;
    s.scalars = (uint32_t *)take(staged ? terms * 32 : 0);
    s.points = (uint32_t *)take(staged ? terms * pin : 0);
    s.digits = (int8_t *)take(terms * (ct ? 64 : NAF_LEN));
    s.tables = (ge_pniels_packed *)take(terms * 8 * sizeof(ge_pniels_packed));
    s.partial = (double *)take(chunks * 20 * sizeof(double));
    s.bytes = at;
}

template <int FMT>
static void mb_launch_fmt(const MbSlot &s, const uint32_t *d_s, const uint32_t *d_p, const uint64_t *d_off, const MbPiece &p, bool ct,
                          bool want_limbs, int *status, cudaStream_t st)
{
    const size_t n = p.t1 - p.t0;
    const uint32_t nseg = (uint32_t)(p.j1 - p.j0);
    if (n) {
        if (ct) {
            k_mb_prepare<FMT, true><<<cdiv(n, MB_THREADS), MB_THREADS, 0, st>>>(d_s, d_p, n, d_off, nseg, p.t0, s.digits, s.tables, s.ok, status);
            k_mb_chunks<true><<<cdiv(p.nchunks, MB_THREADS), MB_THREADS, 0, st>>>(s.digits, s.tables, d_off, s.chunk_base, nseg, p.nchunks, p.t0, s.partial);
        } else {
            k_mb_prepare<FMT, false><<<cdiv(n, MB_THREADS), MB_THREADS, 0, st>>>(d_s, d_p, n, d_off, nseg, p.t0, s.digits, s.tables, s.ok, status);
            k_mb_chunks<false><<<cdiv(p.nchunks, MB_THREADS), MB_THREADS, 0, st>>>(s.digits, s.tables, d_off, s.chunk_base, nseg, p.nchunks, p.t0, s.partial);
        }
    }
    k_mb_finish<FMT><<<cdiv(nseg, MB_THREADS), MB_THREADS, 0, st>>>(s.partial, s.chunk_base, nseg, s.ok, s.out, want_limbs ? s.limbs : nullptr);
}

// the encoding and the limbs of the identity in the convention of a point format
static void mb_identity(int point_fmt, uint8_t *out, uint64_t *limbs)
{
    memset(out, 0, 32);
    if (point_fmt != DALEK_POINTS_RISTRETTO) out[0] = 1;
    if (limbs) { memset(limbs, 0, 160); limbs[5] = 1; limbs[10] = 1; }
}

static int mb_run(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points, int point_fmt, const uint64_t *offsets, bool on_device,
                  size_t m, int constant_time, uint8_t *out, uint64_t *out_limbs, uint8_t *ok)
{
    if (!ctx || (m && (!offsets || !out))) return DALEK_E_INVALID_ARG;
    if (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED && point_fmt != DALEK_POINTS_RISTRETTO) return DALEK_E_INVALID_ARG;
    if (!m) return DALEK_OK;
    const bool ct = constant_time != 0;
    int rc;
    const uint64_t *h_off = offsets;
    std::vector<uint64_t> off_copy;
    if (on_device) {                       // the sizes decide the pieces, the grids and the workspace: 8 bytes per MSM come back
        CUDA_TRY(ctx, cudaSetDevice(ctx->device));
        off_copy.resize(m + 1);
        CUDA_TRY(ctx, cudaMemcpyAsync(off_copy.data(), offsets, (m + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        h_off = off_copy.data();
    }
    if (!mb_offsets_ok(h_off, m)) { ctx->last_error = "offsets must start at 0, not decrease and end below 2^31"; return DALEK_E_INVALID_ARG; }
    const size_t total = (size_t)h_off[m];
    if (total && (!scalars || !points)) return DALEK_E_INVALID_ARG;
    if (ct && !on_device)                  // Scalar invariant #1 (scalar.rs:214-230): bit 255 clear
        for (size_t i = 0; i < total; i++)
            if (scalars[32 * i + 31] & 0x80) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    MbPlan pl;
    mb_plan(pl, h_off, m, ct);
    const size_t pin = msm_point_bytes(point_fmt);
    MbSlot slot[2];
    mb_carve(slot[0], nullptr, pl.max_terms, pl.max_segs, pl.max_chunks, pin, ct, !on_device);
    const size_t ws_bytes = slot[0].bytes;
    const int nslots = pl.pieces.size() > 1 ? 2 : 1;
    DevBuf *mb_ws[2] = {&ctx->ws[WS_MSM_BATCH_0], &ctx->ws[WS_MSM_BATCH_1]};   // the pieces on each of the two streams
    for (int k = 0; k < nslots; k++) {
        if ((rc = ws_reserve(ctx, *mb_ws[k], ws_bytes))) return rc;
        mb_carve(slot[k], (char *)mb_ws[k]->p, pl.max_terms, pl.max_segs, pl.max_chunks, pin, ct, !on_device);
    }
    int *status = slot[0].status;
    cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
    CUDA_TRY(ctx, cudaMemsetAsync(status, 0, 4, ctx->stream));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    for (size_t k = 0; k < pl.pieces.size(); k++) {
        const MbPiece &p = pl.pieces[k];
        const MbSlot &s = slot[k & 1];
        cudaStream_t st = ss[k & 1];
        const size_t n = p.t1 - p.t0, nseg = p.j1 - p.j0;
        const uint32_t *d_s, *d_p;
        const uint64_t *d_off;
        if (on_device) {
            d_s = (const uint32_t *)(scalars + 32 * p.t0);
            d_p = (const uint32_t *)((const uint8_t *)points + pin * p.t0);
            d_off = offsets + p.j0;
        } else {
            CUDA_TRY(ctx, cudaMemcpyAsync(s.offsets, h_off + p.j0, (nseg + 1) * 8, cudaMemcpyHostToDevice, st));
            if (n) {
                CUDA_TRY(ctx, cudaMemcpyAsync(s.scalars, scalars + 32 * p.t0, n * 32, cudaMemcpyHostToDevice, st));
                CUDA_TRY(ctx, cudaMemcpyAsync(s.points, (const uint8_t *)points + pin * p.t0, n * pin, cudaMemcpyHostToDevice, st));
            }
            d_s = s.scalars; d_p = s.points; d_off = s.offsets;
        }
        CUDA_TRY(ctx, cudaMemcpyAsync(s.chunk_base, pl.chunk_base.data() + p.cb, (nseg + 1) * 4, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemsetAsync(s.ok, 1, nseg, st));
        if (point_fmt == DALEK_POINTS_EXTENDED) mb_launch_fmt<DALEK_POINTS_EXTENDED>(s, d_s, d_p, d_off, p, ct, out_limbs != nullptr, status, st);
        else if (point_fmt == DALEK_POINTS_RISTRETTO) mb_launch_fmt<DALEK_POINTS_RISTRETTO>(s, d_s, d_p, d_off, p, ct, out_limbs != nullptr, status, st);
        else mb_launch_fmt<DALEK_POINTS_COMPRESSED>(s, d_s, d_p, d_off, p, ct, out_limbs != nullptr, status, st);
        ctx->launches += n ? 3 : 1;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(out + 32 * p.j0, s.out, nseg * 32, cudaMemcpyDeviceToHost, st));
        if (out_limbs) CUDA_TRY(ctx, cudaMemcpyAsync(out_limbs + 20 * p.j0, s.limbs, nseg * 160, cudaMemcpyDeviceToHost, st));
        if (ok) CUDA_TRY(ctx, cudaMemcpyAsync(ok + p.j0, s.ok, nseg, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (ct)                                // zeroize on drop
        for (int k = 0; k < nslots; k++)
            CUDA_TRY(ctx, cudaMemsetAsync((char *)mb_ws[k]->p + slot[k].secret0, 0, slot[k].bytes - slot[k].secret0, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    int bad = *(const int *)ctx->h_pinned;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)pl.pieces.size();
    for (size_t j : pl.large) {            // variable time only
        const size_t t0 = (size_t)h_off[j], n = (size_t)(h_off[j + 1] - h_off[j]);
        uint64_t *limbs = out_limbs ? out_limbs + 20 * j : nullptr;
        rc = msm_whole(ctx, scalars + 32 * t0, (const uint8_t *)points + pin * t0, on_device, point_fmt, n, out + 32 * j, limbs);
        if (rc != DALEK_OK && rc != DALEK_NONE) return rc;
        if (rc == DALEK_NONE) { bad |= MB_BAD_POINT; mb_identity(point_fmt, out + 32 * j, limbs); }
        if (ok) ok[j] = rc == DALEK_OK;
    }
    if (bad & MB_BAD_SCALAR) { ctx->last_error = "scalar with bit 255 set (Scalar invariant #1)"; return DALEK_E_INVALID_ARG; }
    if ((bad & MB_BAD_POINT) && ct) {
        ctx->last_error = "a point does not decode (multiscalar_mul takes points, not Options)";
        return DALEK_E_INVALID_ARG;
    }
    return (bad & MB_BAD_POINT) ? DALEK_NONE : DALEK_OK;
}

extern "C" {

int dalek_b200_msm_batch(dalek_b200_ctx *ctx, const uint8_t *scalars, const void *points, int point_fmt, const uint64_t *offsets, size_t m,
                         int constant_time, uint8_t *out, uint64_t *out_limbs, uint8_t *ok)
{
    return mb_run(ctx, scalars, points, point_fmt, offsets, false, m, constant_time, out, out_limbs, ok);
}

int dalek_b200_msm_batch_dev(dalek_b200_ctx *ctx, const void *d_scalars, const void *d_points, int point_fmt, const void *d_offsets, size_t m,
                             int constant_time, uint8_t *out, uint64_t *out_limbs, uint8_t *ok)
{
    return mb_run(ctx, (const uint8_t *)d_scalars, d_points, point_fmt, (const uint64_t *)d_offsets, true, m, constant_time, out, out_limbs, ok);
}

}  // extern "C"
