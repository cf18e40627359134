// pieces.h -- host buffers in and out, streamed in pieces over the context's two streams (copy-in -> kernel ->
// copy-out), for batch calls whose items are independent: the PCIe traffic of one piece hides under the arithmetic
// of its neighbours.  Used by the codecs, X25519, hash-to-group, the plain path of verify_each and the double-base batch.
#pragma once
#include <algorithm>
#include <type_traits>

#include "engine.h"

// Per item: optionally a message of the flat layout (msgs + n + 1 offsets, include/dalek_b200.h; offs = NULL: none),
// in_sz bytes of `in` (0: none), optionally in2_sz bytes of a second input `in2`, out_sz bytes of `out` and optionally
// out2_sz bytes of a second output `out2`.  The messages are staged in WS_STAGING_MSGS at their own offsets and the offsets in
// WS_MSG_OFFSETS, the fixed-width inputs in WS_STAGING_IN (first all of `in`, then all of `in2`), the outputs in
// WS_STAGING_OUT.  launch(d_msgs, d_offs, d_in, d_in2, m, d_out, d_out2, stream) enqueues the kernel of one piece of m items
// and returns an engine code; d_offs points at the piece's m + 1 offsets, which stay absolute (d_msgs is the base of the
// whole staged buffer).  A callback that takes one more size_t argument also receives lo, the index of the piece's first
// item in the batch (for per-item data the kernel reads from elsewhere, such as the signer's expanded keys).  Pieces hold `piece` items (0: 2^16 from 2^17 items up, else one piece).  Sets last_kernel_ms
// to the device span of the whole batch, copies included, and last_kernel_launches to the number of pieces.
template <typename Launch>
static int run_pieces(dalek_b200_ctx *ctx, const uint8_t *msgs, const uint64_t *offs, const uint8_t *in, size_t in_sz,
                      const uint8_t *in2, size_t in2_sz, uint8_t *out, size_t out_sz, uint8_t *out2, size_t out2_sz, size_t n,
                      Launch launch, size_t piece = 0)
{
    int rc;
    if (offs) {
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], (n ? (size_t)offs[n] : 0) + 16))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_MSG_OFFSETS], (n + 1) * 8))) return rc;
    }
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * (in_sz + in2_sz)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], std::max<size_t>(1, n) * (out_sz + out2_sz)))) return rc;
    uint8_t *d_msgs = (uint8_t *)ctx->ws[WS_STAGING_MSGS].p, *d_in = (uint8_t *)ctx->ws[WS_STAGING_IN].p, *d_in2 = d_in + n * in_sz;
    uint8_t *d_out = (uint8_t *)ctx->ws[WS_STAGING_OUT].p, *d_out2 = d_out + n * out_sz;
    uint64_t *d_offs = (uint64_t *)ctx->ws[WS_MSG_OFFSETS].p;
    cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    if (!piece) piece = n >= (1u << 17) ? (size_t)1 << 16 : std::max<size_t>(1, n);   // a multiple of 128 * 8
    size_t k = 0;
    for (size_t lo = 0; lo < n; lo += piece, k++) {
        const size_t m = std::min(piece, n - lo);
        cudaStream_t st = ss[k & 1];
        if (offs) {
            const size_t m0 = (size_t)offs[lo], m1 = (size_t)offs[lo + m];
            if (m1 > m0) CUDA_TRY(ctx, cudaMemcpyAsync(d_msgs + m0, msgs + m0, m1 - m0, cudaMemcpyHostToDevice, st));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_offs + lo, offs + lo, (m + 1) * 8, cudaMemcpyHostToDevice, st));
        }
        if (in_sz) CUDA_TRY(ctx, cudaMemcpyAsync(d_in + lo * in_sz, in + lo * in_sz, m * in_sz, cudaMemcpyHostToDevice, st));
        if (in2_sz) CUDA_TRY(ctx, cudaMemcpyAsync(d_in2 + lo * in2_sz, in2 + lo * in2_sz, m * in2_sz, cudaMemcpyHostToDevice, st));
        if constexpr (std::is_invocable_v<Launch &, const uint8_t *, const uint64_t *, const uint8_t *, const uint8_t *, size_t,
                                          uint8_t *, uint8_t *, cudaStream_t, size_t>)
            rc = launch(d_msgs, d_offs + lo, d_in + lo * in_sz, d_in2 + lo * in2_sz, m, d_out + lo * out_sz, d_out2 + lo * out2_sz, st, lo);
        else
            rc = launch(d_msgs, d_offs + lo, d_in + lo * in_sz, d_in2 + lo * in2_sz, m, d_out + lo * out_sz, d_out2 + lo * out2_sz, st);
        if (rc) return rc;
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(out + lo * out_sz, d_out + lo * out_sz, m * out_sz, cudaMemcpyDeviceToHost, st));
        if (out2_sz) CUDA_TRY(ctx, cudaMemcpyAsync(out2 + lo * out2_sz, d_out2 + lo * out2_sz, m * out2_sz, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)k;
    return 0;
}

// clear the staged inputs (WS_STAGING_IN) and results (WS_STAGING_OUT) of a call that handled secrets (zeroize on drop),
// then wait for the stream
static inline int wipe_staging(dalek_b200_ctx *ctx, size_t in_bytes, size_t out_bytes)
{
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_IN].p, 0, in_bytes, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_STAGING_OUT].p, 0, out_bytes, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}
