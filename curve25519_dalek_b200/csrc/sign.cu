// sign.cu -- Ed25519 signing in bulk (ed25519-dalek, RFC 8032 5.1.5 / 5.1.6):
//   SigningKey::from_bytes + verifying_key   signing.rs:106, :171; hazmat.rs:84-99    k_sign_keys
//   ExpandedSecretKey::from_bytes + VerifyingKey::from   hazmat.rs:84-99, verifying.rs:97-102   k_esk_keys
//   Signer::try_sign -> raw_sign             signing.rs:566-571, :854-904; hazmat.rs:137   k_sign<0>
//   sign_prehashed -> raw_sign_prehashed     signing.rs:312, :917-976; hazmat.rs:182 (Ed25519ph)   k_sign<1>
//
// k_sign_keys, one thread per seed: (a, prefix) = SHA-512(seed), a clamped; A = [a]B over the clamped, unreduced a
// (the same point as [a mod l]B), compressed.  k_esk_keys does the same from 64 ExpandedSecretKey bytes, without the hash.
// k_sign, one thread per message: r = SHA-512(prefix || M) mod l
// (Ed25519ph: SHA-512(dom2(1, C) || prefix || PH)), R = [r]B, k = SHA-512(R || A || M) (Ed25519ph: dom2 || R || A || PH)
// mod l, s = k a + r mod l.  Both multiplications by B are the constant-time comb of comb.cuh over the table of B that
// the X25519 public keys use (comb_base_table_ensure), staged in shared memory: 60 KiB, 384 threads, one block per SM.
// k_sign clamps a as it loads it, so the hazmat calls feed the caller's ExpandedSecretKey bytes to it as staged; A is
// then the caller's verifying key, hashed as given.
// With one key for the whole batch every message reads the same expanded key.  A signing-key set keeps its expanded keys
// and verifying keys in device memory of its own, and each message reads the key its index names.
//
// Constant time.  Secrets: the seed, SHA-512(seed), an ExpandedSecretKey, a, prefix, r, k a and s before it is written
// out.  Public: the messages and their lengths, the prehashes, the context, the key indices (which key signs a message
// is not secret in the reference either), A, R, k and the signature.
//   - No branch, loop bound or memory address depends on a secret.  The comb scans all 8 entries of each of its 64 rows
//     and applies the digit's sign by the masked swap / negate of ge64_madd; the radix-16 recoding is arithmetic.
//   - SHA-512 inputs are assembled in registers (hash.cuh, sha512_pxm); which word a byte comes from depends on the
//     lengths of the message and the context only.
//   - Scalars mod l (sc.cuh) are branch-free: the conditional subtractions of l are masked selects.
//   - R and A are encoded with the fixed inversion chain of ge_compress<1> and the branch-free canonical encoding.
//   - The device copies of the seeds, of the ExpandedSecretKey bytes and of the expanded keys (a, prefix) that a call
//     stages are cleared before it returns, failed calls included, as the reference zeroizes them on drop
//     (signing.rs:686-690, hazmat.rs:67-72).  A signing-key set's expanded keys are cleared by its destroy, before the
//     memory is freed.  r, k a and s live in registers, apart from what ptxas spills to the thread's stack frame
//     (DESIGN.md section 9 records the sizes, and tests/test_sign_host.py and tests/test_signing_key_set_host.py hold
//     the kernels to them).
// base.cu's mul_base, which indexes its table by the digit, is not used here.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

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

__device__ __forceinline__ void clamp_scalar(uint32_t a[8])   // clamp_integer (scalar.rs:1407-1412)
{
    a[0] &= 0xfffffff8u;
    a[7] = (a[7] & 0x7fffffffu) | 0x40000000u;
}

// Key i from its 64 expanded bytes h (scalar bytes, then prefix): a = clamp(h[0..8)), kept with the prefix in expanded
// (NULL: not kept), and A = compress([a]B) in pks.  h is consumed.
__device__ __forceinline__ void expanded_key_out(uint32_t h[16], size_t i, uint32_t *__restrict__ expanded,
                                                 uint32_t *__restrict__ pks, const double *s_tab)
{
    clamp_scalar(h);
    if (expanded) {
#pragma unroll
        for (int k = 0; k < 16; k++) expanded[16 * i + k] = h[k];
    }
    uint32_t A[8];
    comb_base_compressed(A, h, s_tab);
#pragma unroll
    for (int k = 0; k < 8; k++) pks[8 * i + k] = A[k];
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
    expanded_key_out(h, i, expanded, pks, s_tab);
}

// esks: n x 16 words of ExpandedSecretKey bytes (the scalar bytes, then hash_prefix), used as given: no seed hash.
// expanded and pks as in k_sign_keys.
__global__ void __launch_bounds__(SIGN_THREADS, 1)
k_esk_keys(const uint32_t *__restrict__ esks, const double *__restrict__ table, size_t n, uint32_t *__restrict__ expanded,
           uint32_t *__restrict__ pks)
{
    extern __shared__ double s_tab[];
    stage_comb_table(s_tab, table);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t h[16];
#pragma unroll
    for (int k = 0; k < 16; k++) h[k] = esks[16 * i + k];
    expanded_key_out(h, i, expanded, pks, s_tab);
}

// PH = 0: message i = msgs[offs[i] .. offs[i+1]) (msgs: the whole staged buffer, offsets absolute); PH = 1: prehash i =
// msgs[64 i .. 64 i + 64), dom = dom2(1, C).  The expanded key and A of message i are entry key_idx[i] of `expanded` /
// `pks` when key_idx is given, else entry key0 + i, or entry 0 for every message when one_key is set.  An index >= nkeys
// is never used as an address: it sets *bad_idx and message i gets 64 zero bytes, never a signature under another key.
// The scalar half of each expanded key is clamped as it is loaded (idempotent on keys clamped already).
// sigs: n x 16 words, R then s.
template <int PH>
__global__ void __launch_bounds__(SIGN_THREADS, 1)
k_sign(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ expanded,
       const uint32_t *__restrict__ pks, size_t key0, int one_key, const uint32_t *__restrict__ key_idx, uint32_t nkeys,
       int *__restrict__ bad_idx, size_t n, const double *__restrict__ table, const __grid_constant__ Sha512Prefix dom,
       uint32_t *__restrict__ sigs)
{
    extern __shared__ double s_tab[];
    stage_comb_table(s_tab, table);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    size_t kk = one_key ? 0 : key0 + i;
    if (key_idx) {                                                // the index is public
        const uint32_t t = key_idx[i];
        if (t >= nkeys) {
            atomicOr(bad_idx, 1);
#pragma unroll
            for (int j = 0; j < 16; j++) sigs[16 * i + j] = 0;
            return;
        }
        kk = t;
    }
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
        clamp_scalar(a);                                          // ExpandedSecretKey::from_bytes (hazmat.rs:84-99)
        sc_mul(ka, k, a);                                         // a < 2^255: the product is below 2^512
        sc_add(s, ka, r);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) { sigs[16 * i + j] = R[j]; sigs[16 * i + 8 + j] = s[j]; }
}

static int sign_attrs(dalek_b200_ctx *ctx)
{
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign_keys, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_esk_keys, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sign<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIGN_SMEM));
    return 0;
}

// the table of B and the kernels' shared-memory limit
static int sign_prepare(dalek_b200_ctx *ctx)
{
    int rc;
    if ((rc = comb_base_table_ensure(ctx))) return rc;
    return sign_attrs(ctx);
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

// Stage n_keys ExpandedSecretKey bytes in WS_VERIFY_HRAM (n_keys x 64 B, secret, clamped by k_sign as it loads them) and
// their verifying keys, as given, in WS_VERIFY_H (n_keys x 32 B), on the main stream: the hazmat calls.
static int stage_expanded(dalek_b200_ctx *ctx, const uint8_t *esks, const uint8_t *vks, size_t n_keys)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_HRAM], n_keys * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_H], n_keys * 32))) return rc;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_VERIFY_HRAM].p, esks, n_keys * 64, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->ws[WS_VERIFY_H].p, vks, n_keys * 32, cudaMemcpyHostToDevice, ctx->stream));
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

// the staged seeds (WS_SCALARS, n_seeds x 32 B) and the expanded keys (WS_VERIFY_HRAM, n_keys x 64 B) of a sign call
static int wipe_keys(dalek_b200_ctx *ctx, size_t n_seeds, size_t n_keys, int rc)
{
    return wipe_secrets(ctx, &ctx->ws[WS_SCALARS], n_seeds * 32, &ctx->ws[WS_VERIFY_HRAM], n_keys * 64, rc);
}

// The keys k_sign reads: nkeys expanded keys (16 words each) and verifying keys (8 words each) in device memory, chosen
// per message by an index (the signing-key sets; bad_idx: their bad-index word), by position, or one for all (one_key).
struct SignKeys {
    const uint32_t *expanded, *pks;
    int one_key;
    uint32_t nkeys;
    int *bad_idx;
};

// one k_sign launch over m messages or prehashes (d_idx: their key indices, device, or NULL)
static void launch_sign(const Sha512Prefix *ph_dom, const uint8_t *d_msgs, const uint64_t *d_offs, const SignKeys &K, size_t key0,
                        const uint32_t *d_idx, size_t m, const double *table, uint8_t *d_out, cudaStream_t st)
{
    if (ph_dom)
        k_sign<1><<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>(d_msgs, nullptr, K.expanded, K.pks, key0, K.one_key, d_idx, K.nkeys,
                                                                         K.bad_idx, m, table, *ph_dom, (uint32_t *)d_out);
    else
        k_sign<0><<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>(d_msgs, d_offs, K.expanded, K.pks, key0, K.one_key, d_idx, K.nkeys,
                                                                         K.bad_idx, m, table, Sha512Prefix{}, (uint32_t *)d_out);
}

// Sign n messages (flat layout, or prehashes when ph_dom is set) from host buffers, streamed in pieces; key_idx (host, n,
// or NULL) travels with the messages.  sigs_out: n x 64 B.
static int sign_pieces(dalek_b200_ctx *ctx, const SignKeys &K, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                       const uint8_t *prehashes, const Sha512Prefix *ph_dom, const uint32_t *key_idx, size_t n, uint8_t *sigs_out)
{
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    const size_t idx_sz = key_idx ? 4 : 0;
    // fixed-width inputs: the prehashes of Ed25519ph, then the key indices
    const uint8_t *in = ph_dom ? prehashes : (const uint8_t *)key_idx, *in2 = ph_dom ? (const uint8_t *)key_idx : nullptr;
    return run_pieces(ctx, ph_dom ? nullptr : msgs_flat, ph_dom ? nullptr : msg_offsets, in, ph_dom ? 64 : idx_sz, in2, ph_dom ? idx_sz : 0,
                      sigs_out, 64, nullptr, 0, n,
                      [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *d_in, const uint8_t *d_in2, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st, size_t key0) {                    // key0: the piece's first item
                          const uint32_t *d_idx = key_idx ? (const uint32_t *)(ph_dom ? d_in2 : d_in) : nullptr;
                          launch_sign(ph_dom, ph_dom ? d_in : d_msgs, d_offs, K, key0, d_idx, m, table, d_o, st);
                          return 0;
                      });
}

// Sign n messages (flat layout, or prehashes when ph_dom is set) with n_keys = n or 1 keys: seeds, expanded on the device
// (vks NULL), or ExpandedSecretKey bytes with their verifying keys (hazmat raw_sign), staged as given.  sigs_out: n x 64 B.
static int sign_common(dalek_b200_ctx *ctx, const uint8_t *keys, const uint8_t *vks, size_t n_keys, const uint8_t *msgs_flat,
                       const uint64_t *msg_offsets, const uint8_t *prehashes, const Sha512Prefix *ph_dom, size_t n,
                       uint8_t *sigs_out)
{
    int rc;
    if ((rc = sign_prepare(ctx))) return rc;
    const size_t n_seeds = vks ? 0 : n_keys;
    if ((rc = vks ? stage_expanded(ctx, keys, vks, n_keys) : expand_keys(ctx, keys, n_keys))) return wipe_keys(ctx, n_seeds, n_keys, rc);
    const SignKeys K{(const uint32_t *)ctx->ws[WS_VERIFY_HRAM].p, (const uint32_t *)ctx->ws[WS_VERIFY_H].p, n_keys == 1, 0, nullptr};
    rc = sign_pieces(ctx, K, msgs_flat, msg_offsets, prehashes, ph_dom, nullptr, n, sigs_out);
    return wipe_keys(ctx, n_seeds, n_keys, rc);
}

// ---- resident signing-key sets ------------------------------------------------------------------------------------------
// A service that signs at volume holds a fixed set of keys.  A set derives its k keys once (k_sign_keys from seeds or
// keypairs, k_esk_keys from ExpandedSecretKey bytes) into device memory of its own, and every later call sends messages
// and key indices only: k_sign reads each message's key by its index, with no key derivation per call.
struct ed25519_b200_signing_key_set {
    dalek_b200_ctx *ctx;   // the context it serves; destroy does not touch it
    int device;
    size_t k;
    uint32_t *d_keys;      // k x 16 words a (clamped) || prefix -- secret -- then k x 8 words A: the layout k_sign reads
    uint8_t *pks;          // host copy of the k x 32 B verifying keys
};

static void signing_key_set_free(ed25519_b200_signing_key_set *s)
{
    if (s->d_keys) {
        cudaMemset(s->d_keys, 0, s->k * 64);                       // zeroize on drop (hazmat.rs:67-72)
        cudaDeviceSynchronize();                                   // the clearing is done and no call still reads the set
        cudaFree(s->d_keys);
    }
    delete[] s->pks;
    delete s;
}

static int signing_key_set_check(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s)
{
    if (!ctx || !s) return DALEK_E_INVALID_ARG;
    if (s->ctx != ctx) { ctx->last_error = "signing-key set used with a context other than its own"; return DALEK_E_INVALID_ARG; }
    return 0;
}

static bool signing_key_indices_ok(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const uint32_t *key_idx, size_t n)
{
    if (key_idx)                                                   // public: checked before any device work
        for (size_t i = 0; i < n; i++)
            if (key_idx[i] >= s->k) { ctx->last_error = "key index >= len()"; return false; }
    return true;
}

// the keys of a set call, with the bad-index word in WS_CALL_SCRATCH cleared on the main stream
static int signing_key_set_keys(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, bool indexed, SignKeys &K)
{
    int rc;
    if ((rc = sign_prepare(ctx))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_CALL_SCRATCH], 4))) return rc;
    int *bad = (int *)ctx->ws[WS_CALL_SCRATCH].p;
    CUDA_TRY(ctx, cudaMemsetAsync(bad, 0, 4, ctx->stream));
    K = SignKeys{s->d_keys, s->d_keys + 16 * s->k, indexed ? 0 : 1, (uint32_t)s->k, bad};
    return 0;
}

extern "C" {

int ed25519_b200_verifying_keys(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n, uint8_t *pubkeys_out)
{
    if (!ctx || (n && (!seeds || !pubkeys_out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = sign_prepare(ctx))) return rc;
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

int ed25519_b200_expanded_verifying_keys(dalek_b200_ctx *ctx, const uint8_t *esks, size_t n, uint8_t *pubkeys_out)
{
    if (!ctx || (n && (!esks || !pubkeys_out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    int rc;
    if ((rc = sign_prepare(ctx))) return rc;
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    rc = run_pieces(ctx, nullptr, nullptr, esks, 64, nullptr, 0, pubkeys_out, 32, nullptr, 0, n,
                    [&](const uint8_t *, const uint64_t *, const uint8_t *d_e, const uint8_t *, size_t m, uint8_t *d_o, uint8_t *,
                        cudaStream_t st) {
                        k_esk_keys<<<cdiv(m, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>((const uint32_t *)d_e, table, m, nullptr,
                                                                                         (uint32_t *)d_o);
                        return 0;
                    });
    return wipe_secrets(ctx, &ctx->ws[WS_STAGING_IN], n * 64, nullptr, 0, rc);                  // the staged esks
}

int ed25519_b200_sign_flat(dalek_b200_ctx *ctx, const uint8_t *seeds, size_t n_seeds, const uint8_t *msgs_flat,
                           const uint64_t *msg_offsets, size_t n, uint8_t *sigs_out)
{
    if (!ctx || (n && (!seeds || !sigs_out)) || (n_seeds != n && n_seeds != 1) || !flat_messages_ok(msgs_flat, msg_offsets, n))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return sign_common(ctx, seeds, nullptr, n_seeds, msgs_flat, msg_offsets, nullptr, nullptr, n, sigs_out);
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
    return sign_common(ctx, seeds, nullptr, n_seeds, nullptr, nullptr, prehashes, &dom, n, sigs_out);
}

int ed25519_b200_raw_sign_flat(dalek_b200_ctx *ctx, const uint8_t *esks, const uint8_t *vks, size_t n_keys, const uint8_t *msgs_flat,
                               const uint64_t *msg_offsets, size_t n, uint8_t *sigs_out)
{
    if (!ctx || (n && (!esks || !vks || !sigs_out)) || (n_keys != n && n_keys != 1) || !flat_messages_ok(msgs_flat, msg_offsets, n))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return sign_common(ctx, esks, vks, n_keys, msgs_flat, msg_offsets, nullptr, nullptr, n, sigs_out);
}

int ed25519_b200_raw_sign_prehashed(dalek_b200_ctx *ctx, const uint8_t *esks, const uint8_t *vks, size_t n_keys,
                                    const uint8_t *prehashes, size_t n, const uint8_t *context, size_t context_len, uint8_t *sigs_out)
{
    if (!ctx || (n && (!esks || !vks || !prehashes || !sigs_out)) || (n_keys != n && n_keys != 1) || (context_len && !context))
        return DALEK_E_INVALID_ARG;
    if (context_len > 255) return ED25519_ERR_PREHASHED_CONTEXT_LENGTH;     // signing.rs:931-933
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    Sha512Prefix dom;
    ed25519ph_dom2(dom, context, context_len);
    return sign_common(ctx, esks, vks, n_keys, nullptr, nullptr, prehashes, &dom, n, sigs_out);
}

int ed25519_b200_signing_key_set_new(dalek_b200_ctx *ctx, const uint8_t *keys, size_t k, int form, uint8_t *status,
                                     ed25519_b200_signing_key_set **out)
{
    if (!ctx || !out) return DALEK_E_INVALID_ARG;
    *out = nullptr;
    if (!keys || !k || k > 0xffffffffull ||
        (form != DALEK_SIGNING_KEY_SEED && form != DALEK_SIGNING_KEY_KEYPAIR && form != DALEK_SIGNING_KEY_EXPANDED))
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    if (status) memset(status, 0, k);
    int rc;
    if ((rc = sign_prepare(ctx))) return rc;
    const size_t in_bytes = form == DALEK_SIGNING_KEY_EXPANDED ? 64 : 32;          // secret bytes per key staged
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], k * in_bytes))) return rc;
    ed25519_b200_signing_key_set *s = new (std::nothrow) ed25519_b200_signing_key_set();
    if (s) s->pks = new (std::nothrow) uint8_t[k * 32];
    auto fail = [&](int code) {
        if (s) signing_key_set_free(s);
        return code;
    };
    if (!s || !s->pks) { ctx->last_error = "out of host memory for the signing-key set"; return fail(DALEK_E_NOMEM); }
    s->ctx = ctx; s->device = ctx->device; s->k = k;
    if (cudaMalloc((void **)&s->d_keys, k * 96) != cudaSuccess) {
        s->d_keys = nullptr;
        (void)cudaGetLastError();
        ctx->last_error = "cudaMalloc failed for the signing-key set";
        return fail(DALEK_E_NOMEM);
    }
    cudaStream_t st = ctx->stream;
    uint8_t *staged = (uint8_t *)ctx->ws[WS_STAGING_IN].p;
    uint32_t *d_exp = s->d_keys, *d_pks = s->d_keys + 16 * k;
    const double *table = (const double *)ctx->ws[WS_COMB_BASE_TABLE].p;
    bool cuda_ok = cudaEventRecord(ctx->ev_a, st) == cudaSuccess &&
                   (form == DALEK_SIGNING_KEY_KEYPAIR                // the seed halves only
                        ? cudaMemcpy2DAsync(staged, 32, keys, 64, 32, k, cudaMemcpyHostToDevice, st)
                        : cudaMemcpyAsync(staged, keys, k * in_bytes, cudaMemcpyHostToDevice, st)) == cudaSuccess;
    if (cuda_ok) {
        if (form == DALEK_SIGNING_KEY_EXPANDED)
            k_esk_keys<<<cdiv(k, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>((const uint32_t *)staged, table, k, d_exp, d_pks);
        else
            k_sign_keys<<<cdiv(k, SIGN_THREADS), SIGN_THREADS, SIGN_SMEM, st>>>((const uint32_t *)staged, table, k, d_exp, d_pks);
        ctx->launches++;
        cuda_ok = cudaGetLastError() == cudaSuccess && cudaEventRecord(ctx->ev_b, st) == cudaSuccess &&
                  cudaMemcpyAsync(s->pks, d_pks, k * 32, cudaMemcpyDeviceToHost, st) == cudaSuccess;
    }
    rc = wipe_secrets(ctx, &ctx->ws[WS_STAGING_IN], k * in_bytes, nullptr, 0, cuda_ok ? 0 : DALEK_E_CUDA);   // and waits
    if (rc) {
        if (!cuda_ok) ctx->last_error = std::string("signing-key set build: ") + cudaGetErrorString(cudaGetLastError());
        return fail(rc);
    }
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = 1;
    if (form == DALEK_SIGNING_KEY_KEYPAIR) {
        // SigningKey::from_keypair_bytes (signing.rs:140-150): VerifyingKey::try_from(public half) first, then byte equality
        // with the derived key (verifying.rs:91-95).  Both halves compared are public.  Only a mismatching public half is
        // decoded, to tell PointDecompression from MismatchedKeypair: a half equal to the derived key decodes.
        std::vector<size_t> bad;
        for (size_t i = 0; i < k; i++)
            if (memcmp(keys + 64 * i + 32, s->pks + 32 * i, 32)) bad.push_back(i);
        if (!bad.empty()) {
            std::vector<uint8_t> enc(bad.size() * 32), ok(bad.size());
            std::vector<uint64_t> limbs(bad.size() * 20);
            for (size_t j = 0; j < bad.size(); j++) memcpy(&enc[32 * j], keys + 64 * bad[j] + 32, 32);
            rc = dalek_b200_edwards_decompress_batch(ctx, enc.data(), bad.size(), limbs.data(), ok.data());
            if (rc < 0) return fail(rc);
            for (size_t j = 0; j < bad.size(); j++)
                if (status) status[bad[j]] = ok[j] ? ED25519_ERR_MISMATCHED_KEYPAIR : ED25519_ERR_POINT_DECOMPRESSION;
            ctx->last_error = ok[0] ? "a keypair's public half is not the key derived from its secret half"
                                    : "a keypair's public half does not decode";
            return fail(ok[0] ? ED25519_ERR_MISMATCHED_KEYPAIR : ED25519_ERR_POINT_DECOMPRESSION);
        }
    }
    *out = s;
    return DALEK_OK;
}

size_t ed25519_b200_signing_key_set_len(const ed25519_b200_signing_key_set *s) { return s ? s->k : 0; }

int ed25519_b200_signing_key_set_verifying_keys(const ed25519_b200_signing_key_set *s, uint8_t *pubkeys_out)
{
    if (!s || !pubkeys_out) return DALEK_E_INVALID_ARG;
    memcpy(pubkeys_out, s->pks, s->k * 32);
    return DALEK_OK;
}

void ed25519_b200_signing_key_set_destroy(ed25519_b200_signing_key_set *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    signing_key_set_free(s);
}

int ed25519_b200_signing_key_set_sign_flat(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const uint8_t *msgs_flat,
                                           const uint64_t *msg_offsets, const uint32_t *key_idx, size_t n, uint8_t *sigs_out)
{
    int rc;
    if ((rc = signing_key_set_check(ctx, s))) return rc;
    if ((n && !sigs_out) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    if (!signing_key_indices_ok(ctx, s, key_idx, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    SignKeys K;
    if ((rc = signing_key_set_keys(ctx, s, key_idx != nullptr, K))) return rc;
    return sign_pieces(ctx, K, msgs_flat, msg_offsets, nullptr, nullptr, key_idx, n, sigs_out);
}

int ed25519_b200_signing_key_set_sign_flat_dev(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const void *d_msgs_flat,
                                               const void *d_msg_offsets, const void *d_key_idx, size_t n, void *d_sigs_out)
{
    int rc;
    if ((rc = signing_key_set_check(ctx, s))) return rc;
    if (n && (!d_msg_offsets || !d_sigs_out)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    SignKeys K;
    if ((rc = signing_key_set_keys(ctx, s, d_key_idx != nullptr, K))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    launch_sign(nullptr, (const uint8_t *)d_msgs_flat, (const uint64_t *)d_msg_offsets, K, 0, (const uint32_t *)d_key_idx, n,
                (const double *)ctx->ws[WS_COMB_BASE_TABLE].p, (uint8_t *)d_sigs_out, st);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, K.bad_idx, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = 1;
    if (*(const int *)ctx->h_pinned) { ctx->last_error = "key index >= len()"; return DALEK_E_INVALID_ARG; }
    return DALEK_OK;
}

int ed25519_b200_signing_key_set_sign_prehashed(dalek_b200_ctx *ctx, const ed25519_b200_signing_key_set *s, const uint8_t *prehashes,
                                                const uint8_t *context, size_t context_len, const uint32_t *key_idx, size_t n,
                                                uint8_t *sigs_out)
{
    int rc;
    if ((rc = signing_key_set_check(ctx, s))) return rc;
    if ((n && (!prehashes || !sigs_out)) || (context_len && !context)) return DALEK_E_INVALID_ARG;
    if (!signing_key_indices_ok(ctx, s, key_idx, n)) return DALEK_E_INVALID_ARG;
    if (context_len > 255) return ED25519_ERR_PREHASHED_CONTEXT_LENGTH;     // signing.rs:931-933
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    Sha512Prefix dom;
    ed25519ph_dom2(dom, context, context_len);
    SignKeys K;
    if ((rc = signing_key_set_keys(ctx, s, key_idx != nullptr, K))) return rc;
    return sign_pieces(ctx, K, nullptr, nullptr, prehashes, &dom, key_idx, n, sigs_out);
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
