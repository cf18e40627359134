// scalars.cu -- scalar batch calls (SURVEY 8f rank 4), over the arithmetic mod l of sc.cuh:
//   Scalar::from_bytes_mod_order_wide     C/scalar.rs:248-250      k_scalar_from_wide
//   Scalar::invert_batch / _alloc         C/scalar.rs:779-853      k_scalar_invert_groups, k_scalar_product
//   Add / Sub / Mul                       C/scalar.rs:317-362      k_scalar_binary<OP>      one thread per item
//   Neg / invert / div_by_2               C/scalar.rs:366-374, :739-741, :858-870
//                                                                  k_scalar_unary<OP>       one thread per item
//   from_bytes_mod_order / from_canonical_bytes
//                                         C/scalar.rs:235-244, :259-263
//                                                                  k_scalar_from_bytes<MODE>
//   hash_from_bytes::<Sha512>             C/scalar.rs:617-670      k_scalar_hash_bytes
//   Sum / Product over segments           C/scalar.rs:454-476      k_scalar_fold_chunks<OP> one CTA per chunk: strided
//                                                                  runs, a warp shuffle tree, a shared-memory tree;
//                                                                  k_scalar_fold_finish<OP> one thread per segment
// The batch inversion uses Montgomery's trick like the reference (scalar.rs:806-850): a thread owns SC_K consecutive
// scalars, so one exponentiation by l - 2 (sc_invert) is shared by SC_K scalars; the product of all inverses that the
// reference returns is the product of the per-thread inverses.
// The arithmetic calls take canonical scalars (< l, Scalar invariant #2) and give canonical results.  Every kernel that
// reads scalars tests them with sc_is_canonical, masked, and reports a non-canonical one by a warp reduction and one
// atomic per warp; the call then returns DALEK_E_INVALID_ARG after the batch ran.  Host buffers stream through run_pieces
// (a broadcast operand staged in WS_CALL_SCRATCH); the fold plans its chunks on the host like the point sum (ps_plan.h).
// Constant time in the scalars: no branch, loop bound or address depends on a value; ops, counts, broadcast and segment
// offsets are public.  Every new call clears the engine's copies of its scalars, intermediates and results before it
// returns, also after a failed launch.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/dalek_b200.h"
#include "elligator.cuh"
#include "engine.h"
#include "pieces.h"
#include "ps_plan.h"
#include "sc.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define SC_K 8

__global__ void k_scalar_from_wide(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[16], r[8];
#pragma unroll
    for (int k = 0; k < 16; k++) x[k] = in[16 * i + k];
    sc_reduce512(r, x);
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * i + k] = r[k];
}

// per thread: inverses of SC_K scalars (reduced mod l first); group_inv[t] = inverse of the group's product;
// *zero_flag set if a scalar is 0 mod l (the reference requires nonzero inputs)
__global__ void __launch_bounds__(128)
k_scalar_invert_groups(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out, uint32_t *__restrict__ group_inv,
                       int *__restrict__ zero_flag)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i0 = t * SC_K;
    if (i0 >= n) return;
    uint32_t v[SC_K][8], scratch[SC_K][8], acc[8], tmp[8];
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = k == 0 ? 1u : 0u;
#pragma unroll
    for (int j = 0; j < SC_K; j++) {
        if (i0 + j < n) {
            uint32_t raw[8];
#pragma unroll
            for (int k = 0; k < 8; k++) raw[k] = in[8 * (i0 + j) + k];
            sc_reduce256(v[j], raw);
            uint32_t nz = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) nz |= v[j][k];
            if (!nz) { atomicOr(zero_flag, 1); v[j][0] = 1; }          // keep the group invertible; the call reports the error
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) v[j][k] = k == 0 ? 1u : 0u;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) scratch[j][k] = acc[k];
        sc_mul(acc, acc, v[j]);
    }
    sc_invert(acc, acc);
#pragma unroll
    for (int k = 0; k < 8; k++) group_inv[8 * t + k] = acc[k];
#pragma unroll
    for (int j = SC_K - 1; j >= 0; j--) {
        sc_mul(tmp, acc, v[j]);
        uint32_t o[8];
        sc_mul(o, acc, scratch[j]);
        if (i0 + j < n) {
#pragma unroll
            for (int k = 0; k < 8; k++) out[8 * (i0 + j) + k] = o[k];
        }
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = tmp[k];
    }
}

// product of `count` scalars (one CTA): strided partial products, then a shared-memory tree
__global__ void __launch_bounds__(256) k_scalar_product(const uint32_t *__restrict__ v, size_t count, uint32_t *__restrict__ out)
{
    __shared__ uint32_t sh[256][8];
    uint32_t acc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = k == 0 ? 1u : 0u;
    for (size_t i = threadIdx.x; i < count; i += blockDim.x) {
        uint32_t x[8];
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] = v[8 * i + k];
        sc_mul(acc, acc, x);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) sh[threadIdx.x][k] = acc[k];
    __syncthreads();
    for (uint32_t d = blockDim.x / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            uint32_t a[8], b[8], r[8];
            for (int k = 0; k < 8; k++) { a[k] = sh[threadIdx.x][k]; b[k] = sh[threadIdx.x + d][k]; }
            sc_mul(r, a, b);
            for (int k = 0; k < 8; k++) sh[threadIdx.x][k] = r[k];
        }
        __syncthreads();
    }
    if (threadIdx.x < 8) out[threadIdx.x] = sh[0][threadIdx.x];
}

// ---- the arithmetic calls ----
#define SC_THREADS 128
#define SC_PIECE ((size_t)1 << 16)          // items per piece of a host-buffer call
#define SC_DEV_PIECE ((size_t)1 << 30)      // items per launch of a device-buffer call
#define SF_CHUNK 1024u                      // scalars (or partials) per chunk of a fold
#define SF_THREADS 128                      // the most threads of a chunk's CTA
#define SF_PIECE (1u << 18)                 // the most scalars per host-buffer piece of a fold, in whole chunks

// WS_CALL_SCRATCH: the non-canonical flag and the two broadcast operands
#define SC_BAD 0
#define SC_BCAST_A 256
#define SC_BCAST_B 512
#define SC_SCRATCH 1024

__device__ __forceinline__ void sc_load(uint32_t x[8], const uint32_t *p)
{
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = p[k];
}

__device__ __forceinline__ void sc_store(uint32_t *p, const uint32_t x[8])
{
#pragma unroll
    for (int k = 0; k < 8; k++) p[k] = x[k];
}

// out[i] = op(A_i, B_i) (a_step / b_step 0 broadcast item 0).  out may be a (or b) exactly: each thread reads its item
// before it writes it, so the pointers are not __restrict__.
template <int OP>
__global__ void __launch_bounds__(SC_THREADS)
k_scalar_binary(const uint32_t *a, size_t a_step, const uint32_t *b, size_t b_step, size_t n, uint32_t *out, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[8], y[8], r[8];
    sc_load(x, a + 8 * a_step * i);
    sc_load(y, b + 8 * b_step * i);
    const uint32_t good = sc_is_canonical(x) & sc_is_canonical(y);
    if (OP == DALEK_SCALAR_ADD) sc_add(r, x, y);
    else if (OP == DALEK_SCALAR_SUB) sc_sub(r, x, y);
    else sc_mul(r, x, y);
    sc_store(out + 8 * i, r);
    warp_report_bad(good, bad);
}

template <int OP>
__global__ void __launch_bounds__(SC_THREADS) k_scalar_unary(const uint32_t *in, size_t n, uint32_t *out, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[8], r[8];
    sc_load(x, in + 8 * i);
    const uint32_t good = sc_is_canonical(x);
    if (OP == DALEK_SCALAR_NEG) sc_neg(r, x);
    else if (OP == DALEK_SCALAR_INVERT) sc_invert(r, x);
    else sc_div_by_2(r, x);
    sc_store(out + 8 * i, r);
    warp_report_bad(good, bad);
}

// MOD_ORDER: any 32 bytes mod l, ok 1.  CANONICAL: the bytes when canonical (ok 1), else zero bytes and ok 0.
template <int MODE>
__global__ void __launch_bounds__(SC_THREADS)
k_scalar_from_bytes(const uint32_t *__restrict__ in, size_t n, uint32_t *__restrict__ out, uint8_t *__restrict__ ok, int *bad)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[8], r[8];
    sc_load(x, in + 8 * i);
    uint32_t good = 1;
    if (MODE == DALEK_SCALAR_MOD_ORDER) {
        sc_reduce256(r, x);
    } else {
        good = sc_is_canonical(x);
        const uint32_t m = 0u - good;
#pragma unroll
        for (int k = 0; k < 8; k++) r[k] = x[k] & m;
    }
    sc_store(out + 8 * i, r);
    if (ok) ok[i] = (uint8_t)good;                      // the pointer is public
    warp_report_bad(good, bad);
}

// Scalar::hash_from_bytes::<Sha512>: SHA-512 of message i, from_bytes_mod_order_wide.  msgs: the whole flat buffer
// (offsets are absolute); offs: this piece's n + 1 offsets.
__global__ void __launch_bounds__(SC_THREADS)
k_scalar_hash_bytes(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, size_t n, uint32_t *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t o0 = offs[i], o1 = offs[i + 1];
    uint32_t w[16], r[8];
    h2c_sha512_digest(w, msgs + o0, (size_t)(o1 - o0));
    sc_reduce512(r, w);
    sc_store(out + 8 * i, r);
}

// ---- Sum / Product ----
template <int OP>
__device__ __forceinline__ void sf_identity(uint32_t acc[8])
{
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = (OP == DALEK_SCALAR_PRODUCT && k == 0) ? 1u : 0u;
}

template <int OP>
__device__ __forceinline__ void sf_fold(uint32_t acc[8], const uint32_t x[8])
{
    if (OP == DALEK_SCALAR_SUM) sc_add(acc, acc, x);
    else sc_mul(acc, acc, x);
}

// acc of lane 0 <- the fold of the accumulators of lanes 0 .. lanes-1 (eight words per shuffle step)
template <int OP>
__device__ __forceinline__ void sf_warp_fold(uint32_t acc[8], uint32_t lanes)
{
    uint32_t x[8];
#pragma unroll 1
    for (uint32_t d = (1u << (32 - __clz((int)(lanes - 1)))) >> 1; d > 0; d >>= 1) {
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] = __shfl_down_sync(0xffffffffu, acc[k], (int)d);
        sf_fold<OP>(acc, x);
    }
}

// chunk c = c0 + blockIdx.x (items start[c] .. start[c+1] of in) -> partial[c].  Thread t folds items t, t + blockDim.x,
// ...; the lanes of each warp are folded by a shuffle tree, the warps through shared memory.  Every bound is the chunk
// length, which is public.  The items are tested for canonicity (partials always pass).
template <int OP>
__global__ void __launch_bounds__(SF_THREADS)
k_scalar_fold_chunks(const uint32_t *__restrict__ in, const uint32_t *__restrict__ start, uint32_t c0, uint32_t *__restrict__ partial,
                     int *bad)
{
    __shared__ uint32_t s_warp[SF_THREADS / 32][8];
    const uint32_t c = c0 + blockIdx.x;
    const uint32_t first = start[c], len = start[c + 1] - start[c];
    uint32_t acc[8], x[8], good = 1;
    sf_identity<OP>(acc);
#pragma unroll 1
    for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) {
        sc_load(x, in + 8 * (size_t)(first + k));
        good &= sc_is_canonical(x);
        sf_fold<OP>(acc, x);
    }
    warp_report_bad(good, bad);
    sf_warp_fold<OP>(acc, len < 32 ? len : 32);
    const uint32_t nw = min((len + 31) / 32, blockDim.x / 32);   // warps that hold items
    if (nw > 1) {
        const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        if (lane == 0) sc_store(s_warp[wid], acc);
        __syncthreads();
        if (wid == 0) {
            if (lane < nw) sc_load(acc, s_warp[lane]);
            else sf_identity<OP>(acc);
            sf_warp_fold<OP>(acc, nw);
        }
    }
    if (threadIdx.x == 0) sc_store(partial + 8 * (size_t)c, acc);
}

// segment j: its one partial, or the identity when it is empty (public)
template <int OP>
__global__ void __launch_bounds__(SC_THREADS)
k_scalar_fold_finish(const uint32_t *__restrict__ partial, const uint32_t *__restrict__ seg_base, size_t m, uint32_t *__restrict__ out)
{
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    uint32_t acc[8];
    sf_identity<OP>(acc);
    if (seg_base[j + 1] > seg_base[j]) sc_load(acc, partial + 8 * (size_t)seg_base[j]);
    sc_store(out + 8 * j, acc);
}

// ---- host side of the arithmetic calls ----
// item counts up to this keep every byte count of a call (64 B per item at most) far from overflow
static bool sc_count_ok(dalek_b200_ctx *ctx, size_t n)
{
    if (n <= (SIZE_MAX >> 8)) return true;
    ctx->last_error = "too many items: the byte counts overflow";
    return false;
}

// Clear what the call left on the device (staged inputs, messages, results, scratch, fold workspace), up to what each
// workspace holds, after reading the non-canonical flag (when the call got that far) into *bad; then wait.  The call's
// result is its first failure, else the wipe's.
static int sc_finish(dalek_b200_ctx *ctx, int rc, size_t in_bytes, size_t out_bytes, size_t msg_bytes, size_t fold_bytes, int *bad)
{
    *bad = 0;
    int *h_bad = (int *)ctx->h_pinned;
    const bool read = !rc && h_bad;
    if (read && cudaMemcpyAsync(h_bad, (char *)ctx->ws[WS_CALL_SCRATCH].p + SC_BAD, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) {
        ctx->last_error = "reading the call's status failed";
        rc = DALEK_E_CUDA;
    }
    auto clear = [&](DevBuf &w, size_t bytes) {
        if (w.p && bytes && cudaMemsetAsync(w.p, 0, std::min(bytes, w.cap), ctx->stream) != cudaSuccess) return false;
        return true;
    };
    bool good = clear(ctx->ws[WS_STAGING_IN], in_bytes) && clear(ctx->ws[WS_STAGING_OUT], out_bytes) &&
                clear(ctx->ws[WS_STAGING_MSGS], msg_bytes) && clear(ctx->ws[WS_CALL_SCRATCH], SC_SCRATCH) &&
                clear(ctx->ws[WS_SCALAR_FOLD], fold_bytes);
    good = cudaStreamSynchronize(ctx->stream) == cudaSuccess && good;
    if (!good && !rc) { ctx->last_error = "clearing the call's device buffers failed"; rc = DALEK_E_CUDA; }
    if (!rc && read) *bad = *h_bad;
    return rc;
}

// launch(a, a_step, b, b_step, m, out, ok, bad, stream) enqueues one piece
typedef void (*ScLaunch)(const uint32_t *, size_t, const uint32_t *, size_t, size_t, uint32_t *, uint8_t *, int *, cudaStream_t);

template <int OP>
static void sc_binary_launch(const uint32_t *a, size_t as, const uint32_t *b, size_t bs, size_t m, uint32_t *out, uint8_t *, int *bad,
                             cudaStream_t st)
{
    k_scalar_binary<OP><<<cdiv(m, SC_THREADS), SC_THREADS, 0, st>>>(a, as, b, bs, m, out, bad);
}

template <int OP>
static void sc_unary_launch(const uint32_t *a, size_t, const uint32_t *, size_t, size_t m, uint32_t *out, uint8_t *, int *bad, cudaStream_t st)
{
    k_scalar_unary<OP><<<cdiv(m, SC_THREADS), SC_THREADS, 0, st>>>(a, m, out, bad);
}

template <int MODE>
static void sc_from_bytes_launch(const uint32_t *a, size_t, const uint32_t *, size_t, size_t m, uint32_t *out, uint8_t *ok, int *bad,
                                 cudaStream_t st)
{
    k_scalar_from_bytes<MODE><<<cdiv(m, SC_THREADS), SC_THREADS, 0, st>>>(a, m, out, ok, bad);
}

// Every element-wise call after its argument checks: n items of 32 B, a and b with steps n_a, n_b in {1, n} (b NULL for the
// unary calls), ok (nullable) one byte per item.  A flagged item makes the call return `flagged`.
static int sc_run(dalek_b200_ctx *ctx, ScLaunch launch, const void *a, size_t n_a, const void *b, size_t n_b, size_t n, void *out,
                  uint8_t *ok, bool on_device, int flagged)
{
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    const bool ba = n_a == 1, bb = b && n_b == 1;
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], SC_SCRATCH))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    char *scratch = (char *)ctx->ws[WS_CALL_SCRATCH].p;
    int *bad = (int *)(scratch + SC_BAD);
    const uint32_t *bcast_a = (const uint32_t *)(scratch + SC_BCAST_A), *bcast_b = (const uint32_t *)(scratch + SC_BCAST_B);
    const size_t a_sz = ba ? 0 : 32, b_sz = (!b || bb) ? 0 : 32, ok_sz = ok ? 1 : 0;
    rc = 0;
    if (cudaMemsetAsync(bad, 0, 4, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
    if (!rc && !on_device) {
        if (ba && cudaMemcpyAsync((void *)bcast_a, a, 32, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        if (bb && cudaMemcpyAsync((void *)bcast_b, b, 32, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        if (!rc)
            rc = run_pieces(ctx, nullptr, nullptr, ba ? nullptr : (const uint8_t *)a, a_sz, b_sz ? (const uint8_t *)b : nullptr, b_sz,
                            (uint8_t *)out, 32, ok, ok_sz, n,
                            [&](const uint8_t *, const uint64_t *, const uint8_t *d_a, const uint8_t *d_b, size_t m, uint8_t *d_o,
                                uint8_t *d_ok, cudaStream_t st) {
                                launch(ba ? bcast_a : (const uint32_t *)d_a, ba ? 0 : 1, bb ? bcast_b : (const uint32_t *)d_b, bb ? 0 : 1, m,
                                       (uint32_t *)d_o, ok ? d_ok : nullptr, bad, st);
                                return 0;
                            },
                            SC_PIECE);
    } else if (!rc) {
        const uint32_t *pa = (const uint32_t *)a, *pb = (const uint32_t *)b;
        if (cudaEventRecord(ctx->ev_a, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        size_t k = 0;
        for (size_t lo = 0; !rc && lo < n; lo += SC_DEV_PIECE, k++) {
            const size_t m = std::min(SC_DEV_PIECE, n - lo);
            launch(pa + (ba ? 0 : 8 * lo), ba ? 0 : 1, pb ? pb + (bb ? 0 : 8 * lo) : nullptr, bb ? 0 : 1, m, (uint32_t *)out + 8 * lo,
                   ok ? ok + lo : nullptr, bad, ctx->stream);
            ctx->launches++;
            if (cudaGetLastError() != cudaSuccess) { ctx->last_error = "kernel launch failed"; rc = DALEK_E_CUDA; break; }
        }
        if (!rc && cudaEventRecord(ctx->ev_b, ctx->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        ctx->last_kernel_launches = (int)k;
    }
    int nbad = 0;
    rc = sc_finish(ctx, rc, on_device ? 0 : n * (a_sz + b_sz), on_device ? 0 : n * (32 + ok_sz), 0, 0, &nbad);
    if (!rc && on_device) {
        float ms = 0.f;
        if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    }
    if (rc) return rc;
    if (nbad && flagged == DALEK_E_INVALID_ARG) ctx->last_error = "a scalar is not canonical (>= l or bit 255 set)";
    return nbad ? flagged : DALEK_OK;
}

static int sc_binary(dalek_b200_ctx *ctx, int op, const void *a, size_t n_a, const void *b, size_t n_b, size_t n, void *out, bool on_device)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    ScLaunch f = op == DALEK_SCALAR_ADD ? sc_binary_launch<DALEK_SCALAR_ADD>
               : op == DALEK_SCALAR_SUB ? sc_binary_launch<DALEK_SCALAR_SUB>
               : op == DALEK_SCALAR_MUL ? sc_binary_launch<DALEK_SCALAR_MUL> : nullptr;
    if (!f) { ctx->last_error = "op must be DALEK_SCALAR_ADD, DALEK_SCALAR_SUB or DALEK_SCALAR_MUL"; return DALEK_E_INVALID_ARG; }
    if (!sc_count_ok(ctx, n)) return DALEK_E_INVALID_ARG;
    if (n && (!a || !b || !out)) return DALEK_E_INVALID_ARG;
    if ((n_a != 1 && n_a != n) || (n_b != 1 && n_b != n)) { ctx->last_error = "n_a and n_b must each be 1 or n"; return DALEK_E_INVALID_ARG; }
    return sc_run(ctx, f, a, n_a, b, n_b, n, out, nullptr, on_device, DALEK_E_INVALID_ARG);
}

static int sc_unary(dalek_b200_ctx *ctx, int op, const void *in, size_t n, void *out, bool on_device)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    ScLaunch f = op == DALEK_SCALAR_NEG ? sc_unary_launch<DALEK_SCALAR_NEG>
               : op == DALEK_SCALAR_INVERT ? sc_unary_launch<DALEK_SCALAR_INVERT>
               : op == DALEK_SCALAR_DIV_BY_2 ? sc_unary_launch<DALEK_SCALAR_DIV_BY_2> : nullptr;
    if (!f) { ctx->last_error = "op must be DALEK_SCALAR_NEG, DALEK_SCALAR_INVERT or DALEK_SCALAR_DIV_BY_2"; return DALEK_E_INVALID_ARG; }
    if (!sc_count_ok(ctx, n)) return DALEK_E_INVALID_ARG;
    if (n && (!in || !out)) return DALEK_E_INVALID_ARG;
    return sc_run(ctx, f, in, n, nullptr, 0, n, out, nullptr, on_device, DALEK_E_INVALID_ARG);
}

// ---- Sum / Product ----
// the device arrays of one fold, carved from WS_SCALAR_FOLD
struct SfSlot {
    std::vector<uint32_t *> start;          // per level: the chunks' first items
    uint32_t *seg_base;                     // the last level's chunk of each segment
    uint32_t *part[2];                      // partials of the even and odd levels
    uint32_t *res;                          // results of a host-buffer call
    size_t bytes;
};

static void sf_carve(SfSlot &s, char *p, const std::vector<PsLevel> &lv, size_t m)
{
    size_t at = 0;
    auto take = [&](size_t b) { char *q = p ? p + at : nullptr; at += (b + 255) & ~(size_t)255; return q; };
    s.start.resize(lv.size());
    for (size_t l = 0; l < lv.size(); l++) s.start[l] = (uint32_t *)take(lv[l].start.size() * 4);
    s.seg_base = (uint32_t *)take((m + 1) * 4);
    for (int k = 0; k < 2; k++) s.part[k] = (uint32_t *)take(lv.size() > (size_t)k ? (lv[k].start.size() - 1) * 32 : 0);
    s.res = (uint32_t *)take(m * 32);
    s.bytes = at;
}

// threads of a chunk's CTA: enough warps for the longest chunk, at most SF_THREADS
static unsigned sf_threads(uint32_t max_len)
{
    return (unsigned)std::min<uint32_t>(SF_THREADS, std::max<uint32_t>(32, (max_len + 31) / 32 * 32));
}

template <int OP>
static int sf_enqueue(dalek_b200_ctx *ctx, const SfSlot &s, const std::vector<PsLevel> &lv, const std::vector<uint32_t> &cuts,
                      const uint8_t *scalars, bool on_device, size_t m, uint32_t *d_res, int *d_bad)
{
    cudaStream_t ss[2] = {ctx->stream, ctx->stream2};
    const uint8_t *staged = (const uint8_t *)ctx->ws[WS_STAGING_IN].p;
    const uint32_t *src = (const uint32_t *)(on_device ? scalars : staged);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, ctx->stream));
    const unsigned thr0 = sf_threads(lv[0].max_len);
    for (size_t k = 0; k + 1 < cuts.size(); k++) {          // level 0: pieces of whole chunks over the two streams
        const uint32_t c0 = cuts[k], c1 = cuts[k + 1], p0 = lv[0].start[c0], p1 = lv[0].start[c1];
        cudaStream_t st = ss[k & 1];
        if (!on_device)
            CUDA_TRY(ctx, cudaMemcpyAsync((void *)(staged + (size_t)p0 * 32), scalars + (size_t)p0 * 32, (size_t)(p1 - p0) * 32,
                                          cudaMemcpyHostToDevice, st));
        k_scalar_fold_chunks<OP><<<c1 - c0, thr0, 0, st>>>(src, s.start[0], c0, s.part[0], d_bad);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->stream2));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    for (size_t l = 1; l < lv.size(); l++) {                  // the partials, until every segment has one
        const uint32_t nch = (uint32_t)lv[l].start.size() - 1;
        k_scalar_fold_chunks<OP><<<nch, sf_threads(lv[l].max_len), 0, ctx->stream>>>(s.part[(l - 1) & 1], s.start[l], 0, s.part[l & 1], d_bad);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    const size_t L = lv.size() - 1;
    k_scalar_fold_finish<OP><<<cdiv(m, SC_THREADS), SC_THREADS, 0, ctx->stream>>>(s.part[L & 1], s.seg_base, m, d_res);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, ctx->stream));
    return 0;
}

static int sf_run(dalek_b200_ctx *ctx, int op, const void *scalars, const uint64_t *offsets, size_t m, void *out, bool on_device)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    if (op != DALEK_SCALAR_SUM && op != DALEK_SCALAR_PRODUCT) {
        ctx->last_error = "op must be DALEK_SCALAR_SUM or DALEK_SCALAR_PRODUCT";
        return DALEK_E_INVALID_ARG;
    }
    if (!sc_count_ok(ctx, m)) return DALEK_E_INVALID_ARG;
    if (m && (!offsets || !out)) return DALEK_E_INVALID_ARG;
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
    const size_t total = (size_t)h_off[m];
    if (total && !scalars) return DALEK_E_INVALID_ARG;
    CallTimer timer(ctx);
    std::vector<PsLevel> lv(1);
    ps_plan_level(lv[0], h_off, m, SF_CHUNK);
    while (lv.back().max_per_seg > 1) {
        PsLevel next;
        ps_plan_level(next, lv.back().base.data(), m, SF_CHUNK);
        lv.push_back(std::move(next));
    }
    std::vector<uint32_t> cuts;
    if (on_device) ps_pieces(cuts, lv[0].start, UINT32_MAX);          // nothing to overlap: one launch
    else ps_pieces(cuts, lv[0].start, SF_PIECE);
    SfSlot s;
    sf_carve(s, nullptr, lv, m);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALAR_FOLD], s.bytes))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], SC_SCRATCH))) return rc;
    if (!on_device && (rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, total) * 32))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    sf_carve(s, (char *)ctx->ws[WS_SCALAR_FOLD].p, lv, m);
    int *d_bad = (int *)((char *)ctx->ws[WS_CALL_SCRATCH].p + SC_BAD);
    uint32_t *d_res = on_device ? (uint32_t *)out : s.res;
    auto body = [&]() -> int {
        CUDA_TRY(ctx, cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
        for (size_t l = 0; l < lv.size(); l++)
            CUDA_TRY(ctx, cudaMemcpyAsync(s.start[l], lv[l].start.data(), lv[l].start.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(s.seg_base, lv.back().base.data(), (m + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        int r = op == DALEK_SCALAR_SUM ? sf_enqueue<DALEK_SCALAR_SUM>(ctx, s, lv, cuts, (const uint8_t *)scalars, on_device, m, d_res, d_bad)
                                       : sf_enqueue<DALEK_SCALAR_PRODUCT>(ctx, s, lv, cuts, (const uint8_t *)scalars, on_device, m, d_res, d_bad);
        if (r) return r;
        if (!on_device) CUDA_TRY(ctx, cudaMemcpyAsync(out, d_res, m * 32, cudaMemcpyDeviceToHost, ctx->stream));
        return 0;
    };
    rc = body();
    int nbad = 0;
    rc = sc_finish(ctx, rc, on_device ? 0 : total * 32, 0, 0, s.bytes, &nbad);
    if (rc) return rc;
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)(cuts.size() - 1);
    if (nbad) { ctx->last_error = "a scalar is not canonical (>= l or bit 255 set)"; return DALEK_E_INVALID_ARG; }
    return DALEK_OK;
}

extern "C" {

int dalek_b200_scalar_from_wide_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n) * 32))) return rc;
    if (n) {
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, in, n * 64, cudaMemcpyHostToDevice, st));
        k_scalar_from_wide<<<cdiv(n, 256), 256, 0, st>>>((const uint32_t *)ctx->ws[WS_STAGING_IN].p, n, (uint32_t *)ctx->ws[WS_SCALARS].p);
        ctx->launches++;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(out, ctx->ws[WS_SCALARS].p, n * 32, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return DALEK_OK;
}

int dalek_b200_scalar_invert_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, uint8_t out_product[32])
{
    if (!ctx || !out_product || (n && (!in || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    int rc;
    cudaStream_t st = ctx->stream;
    const size_t groups = (n + SC_K - 1) / SC_K;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], std::max<size_t>(1, n) * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], std::max<size_t>(1, groups) * 32 + 64))) return rc;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    if ((rc = pinned_reserve(ctx, 256))) return rc;
    uint32_t *d_groups = (uint32_t *)ctx->ws[WS_STAGING_MSGS].p, *d_prod = d_groups + 8 * std::max<size_t>(1, groups);
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->ws[WS_FLAGS].p, 0, FLAG_WORDS * sizeof(int), st));
    if (n) {
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_STAGING_IN].p, in, n * 32, cudaMemcpyHostToDevice, st));
        k_scalar_invert_groups<<<cdiv(groups, 128), 128, 0, st>>>((const uint32_t *)ctx->ws[WS_STAGING_IN].p, n, (uint32_t *)ctx->ws[WS_SCALARS].p, d_groups,
                                                                  (int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS);
        ctx->launches++;
    }
    k_scalar_product<<<1, 256, 0, st>>>(d_groups, groups, d_prod);      // empty input: the empty product, 1
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    int *h_zero = (int *)((char *)ctx->h_pinned + 64);
    if (n) CUDA_TRY(ctx, cudaMemcpyAsync(out, ctx->ws[WS_SCALARS].p, n * 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, d_prod, 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(h_zero, (const int *)ctx->ws[WS_FLAGS].p + FLAG_STATUS, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    if (*h_zero) { ctx->last_error = "invert_batch: a scalar is zero (scalar.rs:796-799: inputs MUST be nonzero)"; return DALEK_E_INVALID_ARG; }
    memcpy(out_product, ctx->h_pinned, 32);
    return DALEK_OK;
}

int dalek_b200_scalar_binary_batch(dalek_b200_ctx *ctx, int op, const uint8_t *a, size_t n_a, const uint8_t *b, size_t n_b, size_t n,
                                   uint8_t *out)
{
    return sc_binary(ctx, op, a, n_a, b, n_b, n, out, false);
}

int dalek_b200_scalar_binary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_a, size_t n_a, const void *d_b, size_t n_b, size_t n,
                                       void *d_out)
{
    return sc_binary(ctx, op, d_a, n_a, d_b, n_b, n, d_out, true);
}

int dalek_b200_scalar_unary_batch(dalek_b200_ctx *ctx, int op, const uint8_t *in, size_t n, uint8_t *out)
{
    return sc_unary(ctx, op, in, n, out, false);
}

int dalek_b200_scalar_unary_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_in, size_t n, void *d_out)
{
    return sc_unary(ctx, op, d_in, n, d_out, true);
}

int dalek_b200_scalar_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, int mode, uint8_t *out, uint8_t *ok)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    if (mode != DALEK_SCALAR_MOD_ORDER && mode != DALEK_SCALAR_CANONICAL) {
        ctx->last_error = "mode must be DALEK_SCALAR_MOD_ORDER or DALEK_SCALAR_CANONICAL";
        return DALEK_E_INVALID_ARG;
    }
    if (!sc_count_ok(ctx, n)) return DALEK_E_INVALID_ARG;
    if (n && (!in || !out)) return DALEK_E_INVALID_ARG;
    ScLaunch f = mode == DALEK_SCALAR_MOD_ORDER ? sc_from_bytes_launch<DALEK_SCALAR_MOD_ORDER> : sc_from_bytes_launch<DALEK_SCALAR_CANONICAL>;
    return sc_run(ctx, f, in, n, nullptr, 0, n, out, ok, false, DALEK_NONE);
}

int dalek_b200_scalar_hash_from_bytes_batch(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, size_t n,
                                            uint8_t *out)
{
    if (!ctx) return DALEK_E_INVALID_ARG;
    if (!sc_count_ok(ctx, n)) return DALEK_E_INVALID_ARG;
    if ((n && !out) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], SC_SCRATCH))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    rc = run_pieces(ctx, msgs_flat, msg_offsets, nullptr, 0, nullptr, 0, out, 32, nullptr, 0, n,
                    [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st) {
                        k_scalar_hash_bytes<<<cdiv(m, SC_THREADS), SC_THREADS, 0, st>>>(d_msgs, d_offs, m, (uint32_t *)d_o);
                        return 0;
                    },
                    SC_PIECE);
    int nbad = 0;
    return sc_finish(ctx, rc, 0, n * 32, (size_t)msg_offsets[n] + 16, 0, &nbad);
}

int dalek_b200_scalar_fold_batch(dalek_b200_ctx *ctx, int op, const uint8_t *scalars, const uint64_t *offsets, size_t m, uint8_t *out)
{
    return sf_run(ctx, op, scalars, offsets, m, out, false);
}

int dalek_b200_scalar_fold_batch_dev(dalek_b200_ctx *ctx, int op, const void *d_scalars, const void *d_offsets, size_t m, void *d_out)
{
    return sf_run(ctx, op, d_scalars, (const uint64_t *)d_offsets, m, d_out, true);
}

}  // extern "C"
