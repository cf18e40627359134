// sign.cu -- Ed25519 signing in bulk (ed25519-dalek, RFC 8032 5.1.5 / 5.1.6):
//   SigningKey::from_bytes + verifying_key   signing.rs:106, :171; hazmat.rs:84-99    k_sign_keys
//   Signer::try_sign -> raw_sign             signing.rs:566-571, :854-904               k_sign<0>
//   sign_prehashed -> raw_sign_prehashed     signing.rs:312, :917-976 (Ed25519ph)        k_sign<1>
//
// k_sign_keys, one thread per seed: (a, prefix) = SHA-512(seed), a clamped; A = [a]B over the clamped, unreduced a
// (the same point as [a mod l]B), compressed.  k_sign, one thread per message: r = SHA-512(prefix || M) mod l
// (Ed25519ph: SHA-512(dom2(1, C) || prefix || PH)), R = [r]B, k = SHA-512(R || A || M) (Ed25519ph: dom2 || R || A || PH)
// mod l, s = k a + r mod l.  Both multiplications by B are the constant-time comb of comb.cuh over the table of B that
// the X25519 public keys use (comb_base_table_ensure), staged in shared memory: 60 KiB, 384 threads, one block per SM.
// With one seed for the whole batch, k_sign_keys runs once and every message reads the same expanded key.
//
// Constant time.  Secrets: the seed, SHA-512(seed), a, prefix, r, k a and s before it is written out.  Public: the
// messages and their lengths, the prehashes, the context, A, R, k and the signature.
//   - No branch, loop bound or memory address depends on a secret.  The comb scans all 8 entries of each of its 64 rows
//     and applies the digit's sign by the masked swap / negate of ge64_madd; the radix-16 recoding is arithmetic.
//   - SHA-512 inputs are assembled in registers (hash.cuh, sha512_pxm); which word a byte comes from depends on the
//     lengths of the message and the context only.
//   - Scalars mod l (sc.cuh) are branch-free: the conditional subtractions of l are masked selects.
//   - R and A are encoded with the fixed inversion chain of ge_compress<1> and the branch-free canonical encoding.
//   - The device copies of the seeds and the expanded keys (a, prefix) are cleared before a call returns, failed calls
//     included, as the reference zeroizes them on drop (signing.rs:686-690, hazmat.rs:67-72).  r, k a and s live in
//     registers, apart from what ptxas spills to the thread's stack frame (DESIGN.md section 9 records the sizes, and
//     tests/test_sign_host.py holds the kernels to them).
// base.cu's mul_base, which indexes its table by the digit, is not used here.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "comb.cuh"
#include "engine.h"
#include "hash.cuh"
#include "pieces.h"
#include "sc.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define SIGN_THREADS 384
#define SIGN_SMEM (COMB_BASE_DOUBLES * sizeof(double))

__device__ __forceinline__ void stage_comb_table(double *s_tab, const double *__restrict__ table)
{
    for (int k = threadIdx.x; k < COMB_BASE_DOUBLES; k += blockDim.x) s_tab[k] = table[k];
    __syncthreads();
}

// compress([s]B); s is consumed
__device__ __forceinline__ void comb_base_compressed(uint32_t out[8], uint32_t s[8], const double *s_tab)
{
    ge64_p3 acc;
    comb_mul_base(acc, s, s_tab);
    ge_p3 P;
    ge64_to_p3(P, acc);
    ge_compress<1>(out, P);
}

// seeds: n x 8 words.  expanded (NULL: not kept): n x 16 words, a (clamped) then prefix.  pks: n x 8 words, A.
__global__ void __launch_bounds__(SIGN_THREADS, 1)
k_sign_keys(const uint32_t *__restrict__ seeds, const double *__restrict__ table, size_t n, uint32_t *__restrict__ expanded,
            uint32_t *__restrict__ pks)
{
    extern __shared__ double s_tab[];
    stage_comb_table(s_tab, table);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t h[16];
    {
        uint32_t seed[8];
#pragma unroll
        for (int k = 0; k < 8; k++) seed[k] = seeds[8 * i + k];
        sha512_pxm<1, 0>(h, nullptr, 0, seed, nullptr, nullptr, 0);
    }
    h[0] &= 0xfffffff8u;                                          // clamp_integer (scalar.rs:1407-1412)
    h[7] = (h[7] & 0x7fffffffu) | 0x40000000u;
    if (expanded) {
#pragma unroll
        for (int k = 0; k < 16; k++) expanded[16 * i + k] = h[k];
    }
    uint32_t A[8];
    comb_base_compressed(A, h, s_tab);
#pragma unroll
    for (int k = 0; k < 8; k++) pks[8 * i + k] = A[k];
}

// PH = 0: message i = msgs[offs[i] .. offs[i+1]) (msgs: the whole staged buffer, offsets absolute); PH = 1: prehash i =
// msgs[64 i .. 64 i + 64), dom = dom2(1, C).  The expanded key and A of message i are entry key0 + i of `expanded` / `pks`,
// or entry 0 for every message when one_key is set.  sigs: n x 16 words, R then s.
template <int PH>
__global__ void __launch_bounds__(SIGN_THREADS, 1)
k_sign(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ expanded,
       const uint32_t *__restrict__ pks, size_t key0, int one_key, size_t n, const double *__restrict__ table,
       const __grid_constant__ Sha512Prefix dom, uint32_t *__restrict__ sigs)
{
    extern __shared__ double s_tab[];
    stage_comb_table(s_tab, table);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t kk = one_key ? 0 : key0 + i;
    const uint8_t *m;
    size_t len;
    if (PH) { m = msgs + 64 * i; len = 64; }
    else { const uint64_t lo = offs[i], hi = offs[i + 1]; m = msgs + lo; len = (size_t)(hi - lo); }
    uint32_t r[8];
    {   // r = SHA-512([dom2 ||] prefix || M) mod l  (raw_sign_byupdate signing.rs:887-893; raw_sign_prehashed :952-960)
        uint32_t pf[8], dig[16];
#pragma unroll
        for (int k = 0; k < 8; k++) pf[k] = expanded[16 * kk + 8 + k];
        if (PH) sha512_pxm<1, 1>(dig, dom.b, dom.len, pf, nullptr, m, len);
        else sha512_pxm<1, 0>(dig, nullptr, 0, pf, nullptr, m, len);
        sc_reduce512(r, dig);
    }
    uint32_t R[8];
    {
        uint32_t t[8];
#pragma unroll
        for (int k = 0; k < 8; k++) t[k] = r[k];
        comb_base_compressed(R, t, s_tab);
    }
    uint32_t s[8];
    {   // k = SHA-512([dom2 ||] R || A || M) mod l, s = k a + r  (signing.rs:895-903; :962-976)
        uint32_t A[8], a[8], dig[16], k[8], ka[8];
#pragma unroll
        for (int j = 0; j < 8; j++) A[j] = pks[8 * kk + j];
        if (PH) sha512_pxm<2, 1>(dig, dom.b, dom.len, R, A, m, len);
        else sha512_ram(dig, R, A, m, len);
        sc_reduce512(k, dig);
#pragma unroll
        for (int j = 0; j < 8; j++) a[j] = expanded[16 * kk + j];
        sc_mul(ka, k, a);                                         // a < 2^255: the product is below 2^512
        sc_add(s, ka, r);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) { sigs[16 * i + j] = R[j]; sigs[16 * i + 8 + j] = s[j]; }
}

static int sign_attrs(dalek_b200_ctx *ctx)
{
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign_keys, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    return 0;
}

// Expand n_seeds seeds into WS_VERIFY_HRAM (n_seeds x 64 B, secret) and their verifying keys into WS_VERIFY_H (n_seeds x 32 B),
// on the main stream; the seeds are staged in WS_SCALARS.
static int expand_keys(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], n_seeds * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_HRAM], n_seeds * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_H], n_seeds * 32))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_SCALARS].p, seeds, n_seeds * 32, cudaMemcpyHostToDevice, ctx->stream));
    k_sign_keys<<<cdiv(n_seeds, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, ctx->stream>>>(
        (const uint32_t *)ctx->ws[WS_SCALARS].p, (const double *)ctx->ws[WS_COMB_BASE_TABLE].p, n_seeds, (uint32_t *)ctx->ws[WS_VERIFY_HRAM].p,
        (uint32_t *)ctx->ws[WS_VERIFY_H].p);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

// zeroize on drop: clear `bytes` bytes of each of the two workspaces (NULL: none) and wait until the clearing is done.  Runs
// after a failed call too: a failed run_pieces returns without joining ctx->stream2, so the second stream is drained first
// and no piece left queued there can read or refill a workspace after it has been cleared.  Returns rc, or a CUDA error
// met here when rc is 0.
static int wipe_secrets(dalek_b200_ctx *ctx, DevBuf *a, size_t a_bytes, DevBuf *b, size_t b_bytes, int rc)
{
    cudaError_t e = cudaStreamSynchronize(ctx->stream2);
    if (a && a->p) cudaMemsetAsync(a->p, 0, std::min(a->cap, a_bytes), ctx->stream);
    if (b && b->p) cudaMemsetAsync(b->p, 0, std::min(b->cap, b_bytes), ctx->stream);
    const cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = e2;
    if (!rc && e != cudaSuccess) {
        ctx->last_error = std::string("wipe_secrets: ") + cudaGetErrorString(e);
        return DALEK_E_CUDA;
    }
    return rc;
}

// the staged seeds (WS_SCALARS) and the expanded keys (WS_VERIFY_HRAM) of expand_keys
static int wipe_keys(dalek_b200_ctx *ctx, size_t n_seeds, int rc)
{
    return wipe_secrets(ctx, &ctx->ws[WS_SCALARS], n_seeds * 32, &ctx->ws[WS_VERIFY_HRAM], n_seeds * 64, rc);
}

// Sign n messages (flat layout, or prehashes when ph_dom is set) with n_seeds = n or 1 keys; sigs_out: n x 64 B.
static int sign_common(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *msgs_flat,
                       const uint64_t *msg_offsets, const uint8_t *prehashes, const Sha512Prefix *ph_dom, size_t n,
                       uint8_t *sigs_out)
{
    int rc;
    if ((rc = comb_base_table_ensure(ctx))) return rc;
    if ((rc = sign_attrs(ctx))) return rc;
    if ((rc = expand_keys(ctx, seeds, n_seeds))) return wipe_keys(ctx, n_seeds, rc);
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    const uint32_t *expanded = (const uint32_t *)ctx->ws[WS_VERIFY_HRAM].p, *pks = (const uint32_t *)ctx->ws[WS_VERIFY_H].p;
    const int one_key = n_seeds == 1;
    Sha512Prefix dom = ph_dom ? *ph_dom : Sha512Prefix{};
    rc = run_pieces(ctx, ph_dom ? nullptr : msgs_flat, ph_dom ? nullptr : msg_offsets, prehashes, ph_dom ? 64 : 0, nullptr, 0,
                    sigs_out, 64, nullptr, 0, n,
                    [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *d_ph, const uint8_t *, size_t m, uint8_t *d_o,
                        uint8_t *, cudaStream_t st, size_t key0) {                    // key0: the piece's first item
                        if (ph_dom)
                            k_sign<1><<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>(d_ph, nullptr, expanded, pks, key0, one_key,
                                                                                             m, table, dom, (uint32_t *)d_o);
                        else
                            k_sign<0><<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>(d_msgs, d_offs, expanded, pks, key0, one_key,
                                                                                             m, table, dom, (uint32_t *)d_o);
                        return 0;
                    });
    return wipe_keys(ctx, n_seeds, rc);
}

extern "C" {

int ed25519_b200_verifying_keys(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n, uint8_t *pubkeys_out)
{
    if (!ctx || (n && (!seeds || !pubkeys_out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = comb_base_table_ensure(ctx))) return rc;
    if ((rc = sign_attrs(ctx))) return rc;
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    rc = run_pieces(ctx, nullptr, nullptr, seeds, 32, nullptr, 0, pubkeys_out, 32, nullptr, 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_s, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st) {
                        k_sign_keys<<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>((const uint32_t *)d_s, table, m, nullptr,
                                                                                          (uint32_t *)d_o);
                        return 0;
                    });
    return wipe_secrets(ctx, &ctx->ws[WS_STAGING_IN], n * 32, nullptr, 0, rc);                  // the staged seeds
}

int ed25519_b200_sign_flat(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *msgs_flat,
                           const uint64_t *msg_offsets, size_t n, uint8_t *sigs_out)
{
    if (!ctx || (n && (!seeds || !sigs_out)) || (n_seeds != n && n_seeds != 1) || !flat_messages_ok(msgs_flat, msg_offsets, n))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return sign_common(ctx, seeds, n_seeds, msgs_flat, msg_offsets, nullptr, nullptr, n, sigs_out);
}

int ed25519_b200_sign_prehashed(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *prehashes, size_t n,
                                const uint8_t *context, size_t context_len, uint8_t *sigs_out)
{
    if (!ctx || (n && (!seeds || !prehashes || !sigs_out)) || (n_seeds != n && n_seeds != 1) || (context_len && !context))
        return DALEK_E_INVALID_ARG;
    if (context_len > 255) return ED25519_ERR_PREHASHED_CONTEXT_LENGTH;     // signing.rs:931-933
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    Sha512Prefix dom;
    ed25519ph_dom2(dom, context, context_len);
    return sign_common(ctx, seeds, n_seeds, nullptr, nullptr, prehashes, &dom, n, sigs_out);
}

// Input synthesis for benchmarks and tests: keys and signatures of n messages in one call, on the signer above.
int ed25519_b200_sign_batch_flat(dalek_b200_ctx *ctx, const uint8_t *seeds, const uint8_t *msgs_flat,
                                 const uint64_t *msg_offsets, size_t n, uint8_t *pubkeys_out, uint8_t *sigs_out)
{
    if (!ctx || (n && (!seeds || !pubkeys_out || !sigs_out)) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    int rc;
    if ((rc = ed25519_b200_verifying_keys(ctx, seeds, n, pubkeys_out))) return rc;
    return ed25519_b200_sign_flat(ctx, seeds, n, msgs_flat, msg_offsets, n, sigs_out);
}

}  // extern "C"
