// pieces.h -- host buffers in and out, streamed in pieces over the context's two streams (copy-in -> kernel ->
// copy-out), for batch calls whose items are independent: the PCIe traffic of one piece hides under the arithmetic
// of its neighbours.  Used by the codecs (codecs.cu) and the X25519 batches (x25519.cu).
#pragma once
#include <algorithm>

#include "engine.h"

// Per item: in_sz bytes of `in`, optionally in2_sz bytes of a second input `in2` (in2_sz = 0: none), out_sz bytes of
// `out` and optionally out2_sz bytes of a second output `out2`.  The inputs are staged in ctx->points_in (first all of
// `in`, then all of `in2`), the outputs in ctx->points.  launch(d_in, d_in2, m, d_out, d_out2, stream) enqueues the
// kernel of one piece of m items.  Sets last_kernel_ms to the device span of the whole batch, copies included.
template <typename Launch>
static int run_pieces(dalek_b200_ctx *ctx, const uint8_t *in, size_t in_sz, const uint8_t *in2, size_t in2_sz, uint8_t *out,
                      size_t out_sz, uint8_t *out2, size_t out2_sz, size_t n, Launch launch)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->points_in, std::max<size_t>(1, n) * (in_sz + in2_sz)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->points, std::max<size_t>(1, n) * (out_sz + out2_sz)))) return rc;
    uint8_t *d_in = (uint8_t *)ctx->points_in.p, *d_in2 = d_in + n * in_sz;
    uint8_t *d_out = (uint8_t *)ctx->points.p, *d_out2 = d_out + n * out_sz;
    cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    const size_t piece = n >= (1u << 17) ? (size_t)1 << 16 : std::max<size_t>(1, n);   // a multiple of 128 * 8
    size_t k = 0;
    for (size_t lo = 0; lo < n; lo += piece, k++) {
        const size_t m = std::min(piece, n - lo);
        cudaStream_t st = ss[k & 1];
        CUDA_TRY(ctx, cudaMemcpyAsync(d_in + lo * in_sz, in + lo * in_sz, m * in_sz, cudaMemcpyHostToDevice, st));
        if (in2_sz) CUDA_TRY(ctx, cudaMemcpyAsync(d_in2 + lo * in2_sz, in2 + lo * in2_sz, m * in2_sz, cudaMemcpyHostToDevice, st));
        launch(d_in + lo * in_sz, d_in2 + lo * in2_sz, m, d_out + lo * out_sz, d_out2 + lo * out2_sz, st);
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
