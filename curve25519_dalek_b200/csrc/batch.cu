// batch.cu -- ed25519_dalek::verify_batch (ed25519-dalek/src/batch.rs:146-251) on one H100.
//
//   k_hram        one thread per signature: SHA-512(R || A || M) (batch.rs:179-191), h_i = hash mod l
//                 (batch.rs:213-216), canonical-s check (batch.rs:208-211, signature.rs:89-94)
//   k_transcript  the Merlin transcript of batch.rs:168-205 and the 16-byte z_i draws of batch.rs:219-222: ONE transcript
//                 over the whole batch (the reference's, default) or -- opt-in `verify_chunk` -- one thread per chunk
//   k_coeffs      one thread per signature: z_i*s_i and z_i*h_i mod l (batch.rs:225-233)
//   k_sum_*       B_coefficient = sum z_i s_i, negated (batch.rs:225-230, :241)
//   k_prep_*      R_i / A_i decompression (batch.rs:235-236, verifying.rs:167-175) into Niels form
//   then the (2n+1)-term bucket MSM of msm.cu (batch.rs:240-244) and the identity test (:246-250).
//
// HBM layout: signatures n x 64 B (R || s), keys n x 32 B, messages back to back with n+1 u64
// offsets; hrams n x 64 B; scalars (2n+1) x 32 B = [-sum z_i s_i, z_1..z_n, z_1 h_1..z_n h_n];
// points (2n+1) x 96 B Niels = [B, R_1..R_n, A_1..A_n]  (same order as batch.rs:240-244).
#include <algorithm>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "hash.cuh"
#include "sc.cuh"
#include "transcript_warp.cuh"
#include "ge64.cuh"
#include "warp4_f64.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

__global__ void __launch_bounds__(128)
k_hram(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ sigs,
       const uint32_t *__restrict__ keys, size_t n, uint32_t *__restrict__ hrams, uint32_t *__restrict__ hs,
       int *__restrict__ flags, uint8_t *__restrict__ bad_s)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t R[8], A[8], s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { R[k] = sigs[16 * i + k]; s[k] = sigs[16 * i + 8 + k]; A[k] = keys[8 * i + k]; }
    uint32_t dig[16];
    {
        const uint64_t lo = offs[i], hi = offs[i + 1];
        sha512_ram(dig, R, A, msgs + lo, (size_t)(hi - lo));
    }
#pragma unroll
    for (int k = 0; k < 16; k++) hrams[16 * i + k] = dig[k];
    uint32_t h[8];
    sc_reduce512(h, dig);
#pragma unroll
    for (int k = 0; k < 8; k++) hs[8 * i + k] = h[k];
    if (!sc_is_canonical(s)) { atomicOr(&flags[FLAG_BAD_S], 1); bad_s[i] = 1; }
}

// k_hram for Ed25519ph (verifying.rs:530-535): SHA-512(dom2(1, C) || R || A || PH) with PH the fixed 64-byte prehash
__global__ void __launch_bounds__(128)
k_hram_ph(const uint8_t *__restrict__ phs, const __grid_constant__ Sha512Prefix dom, const uint32_t *__restrict__ sigs,
          const uint32_t *__restrict__ keys, size_t n, uint32_t *__restrict__ hrams, uint32_t *__restrict__ hs,
          int *__restrict__ flags, uint8_t *__restrict__ bad_s)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t R[8], A[8], s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { R[k] = sigs[16 * i + k]; s[k] = sigs[16 * i + 8 + k]; A[k] = keys[8 * i + k]; }
    uint32_t dig[16];
    sha512_pxm<2, 1>(dig, dom.b, dom.len, R, A, phs + 64 * i, 64);
#pragma unroll
    for (int k = 0; k < 16; k++) hrams[16 * i + k] = dig[k];
    uint32_t h[8];
    sc_reduce512(h, dig);
#pragma unroll
    for (int k = 0; k < 8; k++) hs[8 * i + k] = h[k];
    if (!sc_is_canonical(s)) { atomicOr(&flags[FLAG_BAD_S], 1); bad_s[i] = 1; }
}

__global__ void __launch_bounds__(64)
k_transcript(const uint32_t *__restrict__ hrams, const uint32_t *__restrict__ sigs, size_t n, uint32_t chunk,
             uint32_t *__restrict__ zs)
{
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t lo = t * chunk;
    if (lo >= n) return;
    size_t hi = min(lo + (size_t)chunk, n);
    strobe128 s;
    strobe_init(s, (const uint8_t *)"Merlin v1.0", 11);                                  // batch.rs:44, transcript.rs:56
    {   // append_message(b"dom-sep", b"ed25519 batch verification")  (transcript.rs:58, batch.rs:168)
        const uint8_t *lab = (const uint8_t *)"dom-sep";
        const uint8_t *msg = (const uint8_t *)"ed25519 batch verification";
        strobe_begin_op(s, SFLAG_M | SFLAG_A);
        for (int k = 0; k < 7; k++) strobe_absorb_byte(s, lab[k]);
        strobe_absorb_byte(s, 26); strobe_absorb_byte(s, 0); strobe_absorb_byte(s, 0); strobe_absorb_byte(s, 0);
        strobe_begin_op(s, SFLAG_A);
        for (int k = 0; k < 26; k++) strobe_absorb_byte(s, msg[k]);
    }
    for (size_t i = lo; i < hi; i++) merlin_append_words(s, (const uint8_t *)"hram", 4, hrams + 16 * i, 64);      // batch.rs:195-197
    for (size_t i = lo; i < hi; i++) merlin_append_words(s, (const uint8_t *)"sig.s", 5, sigs + 16 * i + 8, 32);  // batch.rs:199-201
    // build_rng().finalize(&mut ZeroRng): meta_ad("rng"), key(32 zero bytes)  (transcript.rs:157-173)
    strobe_begin_op(s, SFLAG_M | SFLAG_A);
    strobe_absorb_byte(s, 'r'); strobe_absorb_byte(s, 'n'); strobe_absorb_byte(s, 'g');
    strobe_begin_op(s, SFLAG_A | SFLAG_C);
    for (int k = 0; k < 32; k++) { strobe_set_byte(s, s.pos, 0); if (++s.pos == STROBE_R) strobe_run_f(s); }
    for (size_t i = lo; i < hi; i++) {
        // TranscriptRng::try_fill_bytes(16): meta_ad(16u32), prf(16)  (transcript.rs:200-206)
        strobe_begin_op(s, SFLAG_M | SFLAG_A);
        strobe_absorb_byte(s, 16); strobe_absorb_byte(s, 0); strobe_absorb_byte(s, 0); strobe_absorb_byte(s, 0);
        strobe_begin_op(s, SFLAG_I | SFLAG_A | SFLAG_C);
        uint32_t z[4] = {0, 0, 0, 0};
        for (int k = 0; k < 16; k++) {
            z[k >> 2] |= strobe_get_byte(s, s.pos) << (8 * (k & 3));
            strobe_set_byte(s, s.pos, 0);
            if (++s.pos == STROBE_R) strobe_run_f(s);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) zs[4 * i + k] = z[k];
    }
}

// The same transcripts, ONE WARP each (transcript_warp.cuh: the Keccak state spread over 25 lanes, the absorbed byte
// stream in closed form): about four times less latency per permutation than one thread.  Used when there are few
// transcripts (a lone sponge is latency-bound); many transcripts keep one thread each (throughput-bound).
__global__ void __launch_bounds__(32)
k_transcript_warp(const uint32_t *__restrict__ hrams, const uint32_t *__restrict__ sigs, size_t n, uint32_t chunk, uint32_t *__restrict__ zs)
{
    const size_t lo = (size_t)blockIdx.x * chunk;
    if (lo >= n) return;
    const size_t hi = min(lo + (size_t)chunk, n);
    merlin_zs_warp(hrams + 16 * lo, sigs + 16 * lo, hi - lo, zs + 4 * lo);
}

// One thread per transcript again (many transcripts: throughput-bound), without per-byte work on the sponge state: the
// absorbed bytes of the current 166-byte rate block are first laid out in a per-thread shared-memory buffer (byte, 16-bit
// or 32-bit stores, whatever the block position allows; the 43-word stride keeps a warp's lock-step stores on 32 different
// banks), then XORed into the state 64 bits at a time with static indices, so the 25 state words never need dynamic
// addressing.  The transcript starts from the constant state after Transcript::new (MERLIN_PREFIX_*, transcript_warp.cuh)
// and the challenge phase (meta_ad + prf per signature) only ever touches bytes 16..41 and 167 of the block: static too.
// Same byte stream as k_transcript (hash.cuh's strobe_* functions), checked against it and the oracle in the tests.
#define TB_WORDS 43u
__global__ void __launch_bounds__(64)
k_transcript_blocks(const uint32_t *__restrict__ hrams, const uint32_t *__restrict__ sigs, size_t n, uint32_t chunk, uint32_t *__restrict__ zs)
{
    __shared__ uint32_t s_buf[64 * TB_WORDS];
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t lo = t * chunk;
    if (lo >= n) return;
    const size_t hi = min(lo + (size_t)chunk, n);
    uint32_t *bw = s_buf + TB_WORDS * threadIdx.x;
    uint8_t *bb = reinterpret_cast<uint8_t *>(bw);
    uint16_t *bh = reinterpret_cast<uint16_t *>(bw);
#pragma unroll
    for (uint32_t w = 0; w < 42; w++) bw[w] = 0;
    uint64_t st[25];
#pragma unroll
    for (int i = 0; i < 25; i++) st[i] = merlin_prefix_lane((uint32_t)i);
    uint32_t pos = MERLIN_PREFIX_POS, pos_begin = MERLIN_PREFIX_POS_BEGIN;
    auto run_f = [&]() {                                                // strobe_run_f with the block's bytes still in the buffer
        bb[pos] ^= (uint8_t)pos_begin; bb[pos + 1] ^= 0x04; bb[STROBE_R + 1] ^= 0x80;
#pragma unroll
        for (int w = 0; w < 21; w++) { st[w] ^= (uint64_t)bw[2 * w] | ((uint64_t)bw[2 * w + 1] << 32); bw[2 * w] = 0; bw[2 * w + 1] = 0; }
        keccak_f1600(st);
        pos = 0; pos_begin = 0;
    };
    auto put = [&](uint32_t v) { bb[pos] = (uint8_t)v; if (++pos == STROBE_R) run_f(); };
    auto put_word = [&](uint32_t w) {                                   // four data bytes, little-endian
        if (pos + 4 < STROBE_R && (pos & 1) == 0) {                     // stays inside the block (166 = 2 mod 4: never ends exactly on it)
            if (pos & 2) { bh[pos >> 1] = (uint16_t)w; bh[(pos >> 1) + 1] = (uint16_t)(w >> 16); } else bw[pos >> 2] = w;
            pos += 4;
        } else {
            put(w & 0xff); put((w >> 8) & 0xff); put((w >> 16) & 0xff); put(w >> 24);
        }
    };
    auto begin_op = [&](uint32_t flags) { const uint32_t old = pos_begin; pos_begin = pos + 1; put(old); put(flags); };
    // (every put site carries an inlined copy of run_f: large code, but measured faster than one shared out-of-line copy)
    for (size_t i = lo; i < hi; i++) {                                  // append_message(b"hram", ..)  batch.rs:195-197
        begin_op(SFLAG_M | SFLAG_A);
        put('h'); put('r'); put('a'); put('m'); put(64); put(0); put(0); put(0);
        begin_op(SFLAG_A);
        const uint4 *src = reinterpret_cast<const uint4 *>(hrams + 16 * i);
#pragma unroll 1
        for (int q = 0; q < 4; q++) { const uint4 v = src[q]; put_word(v.x); put_word(v.y); put_word(v.z); put_word(v.w); }
    }
    for (size_t i = lo; i < hi; i++) {                                  // append_message(b"sig.s", ..)  batch.rs:199-201
        begin_op(SFLAG_M | SFLAG_A);
        put('s'); put('i'); put('g'); put('.'); put('s'); put(32); put(0); put(0); put(0);
        begin_op(SFLAG_A);
        const uint4 *src = reinterpret_cast<const uint4 *>(sigs + 16 * i + 8);
#pragma unroll 1
        for (int q = 0; q < 2; q++) { const uint4 v = src[q]; put_word(v.x); put_word(v.y); put_word(v.z); put_word(v.w); }
    }
    // build_rng().finalize(&mut ZeroRng): meta_ad("rng"), KEY(32 zero bytes)  (transcript.rs:157-173)
    begin_op(SFLAG_M | SFLAG_A);
    put('r'); put('n'); put('g');
    begin_op(SFLAG_A | SFLAG_C);
    if (pos != 0) run_f();
    st[0] = 0; st[1] = 0; st[2] = 0; st[3] = 0;                         // KEY overwrites state bytes 0..31; pos = 32
    // per signature: meta_ad(16u32), prf(16)  (transcript.rs:200-206).  Block bytes P..P+7 = 0, 0x12, 16, 0, 0, 0, P+1, 0x07,
    // run_f at P+8 (st[P+8] ^= P+7, st[P+9] ^= 0x04, st[167] ^= 0x80); P = 32 for the first draw, 16 afterwards
    bool first = true;
#pragma unroll 1
    for (size_t i = lo; i < hi; i++) {
        const uint32_t P = first ? 32u : 16u;
        const uint64_t w0 = ((uint64_t)0x12 << 8) | ((uint64_t)16 << 16) | ((uint64_t)(P + 1) << 48) | ((uint64_t)0x07 << 56);
        const uint64_t w1 = (uint64_t)(P + 7) | ((uint64_t)0x04 << 8);
        if (first) { st[4] ^= w0; st[5] ^= w1; } else { st[2] ^= w0; st[3] ^= w1; }
        st[20] ^= (uint64_t)0x80 << 56;
        keccak_f1600(st);
        zs[4 * i] = (uint32_t)st[0]; zs[4 * i + 1] = (uint32_t)(st[0] >> 32);
        zs[4 * i + 2] = (uint32_t)st[1]; zs[4 * i + 3] = (uint32_t)(st[1] >> 32);
        st[0] = 0; st[1] = 0;
        first = false;
    }
}

#define TRANSCRIPT_WARP_MAX 2048          // up to this many transcripts per launch: one warp each
static void launch_transcripts(dalek_b200_ctx *ctx, cudaStream_t st, const uint32_t *hrams, const uint32_t *sigs, size_t cnt, uint32_t chunk,
                               uint32_t *zs)
{
    const size_t ntr = (cnt + chunk - 1) / chunk;
    if (ntr <= TRANSCRIPT_WARP_MAX && ctx->opt_transcript_warp)
        k_transcript_warp<<<(unsigned)ntr, 32, 0, st>>>(hrams, sigs, cnt, chunk, zs);
    else if (ctx->opt_transcript_blocks)
        k_transcript_blocks<<<cdiv(ntr, 64), 64, 0, st>>>(hrams, sigs, cnt, chunk, zs);
    else
        k_transcript<<<cdiv(ntr, 64), 64, 0, st>>>(hrams, sigs, cnt, chunk, zs);
    ctx->launches++;
}

// out_z[i] = z_i (MSM scalar of R_i), out_zh[i] = z_i h_i (MSM scalar of A_i, or -- with key merging -- the
// summand of its key; may alias hs), zs_prod[i] = z_i s_i
__global__ void __launch_bounds__(128)
k_coeffs(const uint32_t *__restrict__ zs, const uint32_t *__restrict__ sigs, const uint32_t *hs, size_t n,
         uint32_t *__restrict__ out_z, uint32_t *out_zh, uint32_t *__restrict__ zs_prod)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t z[8], s[8], h[8], r[8];
#pragma unroll
    for (int k = 0; k < 4; k++) { z[k] = zs[4 * i + k]; z[4 + k] = 0; }
#pragma unroll
    for (int k = 0; k < 8; k++) { s[k] = sigs[16 * i + 8 + k]; h[k] = hs[8 * i + k]; }
#pragma unroll
    for (int k = 0; k < 8; k++) out_z[8 * i + k] = z[k];
    sc_mul(r, z, h);
#pragma unroll
    for (int k = 0; k < 8; k++) out_zh[8 * i + k] = r[k];
    sc_mul(r, z, s);
#pragma unroll
    for (int k = 0; k < 8; k++) zs_prod[8 * i + k] = r[k];
}

// plain multiword sums (values < l, at most 2^31 of them: 9 words are enough)
__global__ void k_sum_partial(const uint32_t *__restrict__ v, size_t n, uint32_t nthreads, uint32_t *__restrict__ partial)
{
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nthreads) return;
    uint32_t acc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) acc[k] = 0;
    for (size_t i = t; i < n; i += nthreads) {
        uint64_t carry = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { uint64_t x = (uint64_t)acc[k] + v[8 * i + k] + carry; acc[k] = (uint32_t)x; carry = x >> 32; }
        acc[8] += (uint32_t)carry;
    }
#pragma unroll
    for (int k = 0; k < 9; k++) partial[9 * t + k] = acc[k];
}

__global__ void k_sum_final(const uint32_t *__restrict__ partial, uint32_t count, uint32_t *__restrict__ scalars0)
{
    __shared__ uint32_t sh[256][10];
    uint32_t acc[10];
#pragma unroll
    for (int k = 0; k < 10; k++) acc[k] = 0;
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) {
        uint64_t carry = 0;
#pragma unroll
        for (int k = 0; k < 9; k++) { uint64_t x = (uint64_t)acc[k] + partial[9 * i + k] + carry; acc[k] = (uint32_t)x; carry = x >> 32; }
        acc[9] += (uint32_t)carry;
    }
#pragma unroll
    for (int k = 0; k < 10; k++) sh[threadIdx.x][k] = acc[k];
    __syncthreads();
    for (uint32_t d = blockDim.x / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            uint64_t carry = 0;
            for (int k = 0; k < 10; k++) {
                uint64_t x = (uint64_t)sh[threadIdx.x][k] + sh[threadIdx.x + d][k] + carry;
                sh[threadIdx.x][k] = (uint32_t)x; carry = x >> 32;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t x[16], r[8], neg[8];
        for (int k = 0; k < 16; k++) x[k] = k < 10 ? sh[0][k] : 0;
        sc_reduce512(r, x);
        sc_neg(neg, r);                                   // -B_coefficient (batch.rs:241)
        for (int k = 0; k < 8; k++) scalars0[k] = neg[k];
    }
}

// decompress R_i (first half of each signature) of `cnt` signatures into out_R = &points[1 + i0];
// thread cnt writes the basepoint into out_B (slot 0) when given
#ifndef PREP_MIN_BLOCKS
#define PREP_MIN_BLOCKS 3
#endif
template <int F64>
__global__ void __launch_bounds__(128, PREP_MIN_BLOCKS)
k_prep_R(const uint32_t *__restrict__ sigs, size_t cnt, ge_niels_packed *__restrict__ out_R, ge_niels_packed *__restrict__ out_B,
         int *__restrict__ flags, uint8_t *__restrict__ bad_r)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j > cnt || (j == cnt && !out_B)) return;
    fe x, y;
    ge_niels_packed *dst;
    if (j == cnt) {
        fe_const_base_x(x); fe_const_base_y(y);
        dst = out_B;
    } else {
        uint32_t s[8];
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = sigs[16 * j + k];
        dst = out_R + j;
        if (!ge_decompress_affine<F64>(x, y, s)) { atomicOr(&flags[FLAG_BAD_R], 1); bad_r[j] = 1; fe_0(x); fe_1(y); }
    }
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    ge_niels_packed p; ge_niels_pack(p, nl);
    uint4 *o = reinterpret_cast<uint4 *>(dst);
#pragma unroll
    for (int k = 0; k < 6; k++) o[k] = make_uint4(p.w[4 * k], p.w[4 * k + 1], p.w[4 * k + 2], p.w[4 * k + 3]);
}

// Public keys repeat in real batches (the reference's VerifyingKey even carries its decompressed
// point, E/verifying.rs:65-71, so verify_batch never decompresses A at all).  Keys are de-duplicated
// with an open-addressing table of signature indices: the first signature that inserts a key becomes
// its representative and is appended to `uniq` (position = the key's dense id); only representatives are
// decompressed, and the MSM gets ONE term per distinct key whose scalar is the sum of the z_i h_i of its
// signatures -- the same group equation as batch.rs:240-244 with equal points collected.
__global__ void __launch_bounds__(256)
k_key_dedupe(const uint32_t *__restrict__ keys /* all n keys */, size_t i0, size_t cnt, uint32_t *__restrict__ table,
             uint32_t tmask, uint32_t *__restrict__ rep, uint32_t *__restrict__ uniq, uint32_t *__restrict__ dense,
             uint32_t *__restrict__ uniq_count, uint4 hash_seed)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= cnt) return;
    const uint32_t i = (uint32_t)(i0 + j);
    uint32_t k[8];
#pragma unroll
    for (int q = 0; q < 8; q++) k[q] = keys[8 * (size_t)i + q];
    // keyed per context (hash_seed is drawn at dalek_b200_init): the slot sequence of attacker-chosen key bytes cannot be
    // predicted, so crafted keys cannot be made to pile up in one probe run
    uint32_t h = hash_seed.x;
#pragma unroll
    for (int q = 0; q < 8; q++) { h = (h ^ k[q]) * 0x9E3779B1u; h ^= h >> 15; h += (q & 1) ? hash_seed.y : hash_seed.z; }
    h = (h ^ hash_seed.w) * 0x85EBCA77u;
    h ^= h >> 13;
    uint32_t slot = h & tmask;
    for (;;) {
        uint32_t cur = atomicCAS(&table[slot], 0xffffffffu, i);
        if (cur == 0xffffffffu) {                              // first holder of this key
            rep[i] = i;
            uint32_t pos = atomicAdd(uniq_count, 1u);
            uniq[pos] = i; dense[i] = pos;
            return;
        }
        uint32_t diff = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) diff |= keys[8 * (size_t)cur + q] ^ k[q];
        if (diff == 0) { rep[i] = cur; return; }
        slot = (slot + 1) & tmask;
    }
}

// decompress the keys listed in uniq[*lo .. *hi) into points_A[position] (or, without a list, keys
// i0 .. i0+cnt into points_A[index])
template <int F64>
__global__ void __launch_bounds__(128, PREP_MIN_BLOCKS)
k_prep_A(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ uniq, const uint32_t *__restrict__ lo,
         const uint32_t *__restrict__ hi, size_t i0, size_t cnt, ge_niels_packed *__restrict__ points_A, int *__restrict__ flags,
         uint8_t *__restrict__ bad_key /* by slot */)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t i, slot;
    if (uniq) { slot = *lo + j; if (slot >= *hi) return; i = uniq[slot]; } else { if (j >= cnt) return; i = slot = i0 + j; }
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = keys[8 * i + k];
    fe x, y;
    if (!ge_decompress_affine<F64>(x, y, s)) { atomicOr(&flags[FLAG_BAD_A], 1); bad_key[slot] = 1; fe_0(x); fe_1(y); }
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    ge_niels_packed p; ge_niels_pack(p, nl);
    uint4 *o = reinterpret_cast<uint4 *>(points_A + slot);
#pragma unroll
    for (int k = 0; k < 6; k++) o[k] = make_uint4(p.w[4 * k], p.w[4 * k + 1], p.w[4 * k + 2], p.w[4 * k + 3]);
}

// The reference's VerifyingKey already carries its decompressed point (E/verifying.rs:65-71) and verify_batch uses it
// directly (batch.rs:236-238): when the caller passes those points (20 u64 radix-2^51 limbs X | Y | Z | T each) no key
// is decompressed here.  Z = 1 (what VerifyingKey::from_bytes produces) costs nothing; another Z costs one inversion.
template <int F64>
__global__ void __launch_bounds__(128, PREP_MIN_BLOCKS)
k_prep_A_points(const uint64_t *__restrict__ key_points, const uint32_t *__restrict__ uniq, const uint32_t *__restrict__ lo,
                const uint32_t *__restrict__ hi, size_t i0, size_t cnt, ge_niels_packed *__restrict__ points_A)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t i, slot;
    if (uniq) { slot = *lo + j; if (slot >= *hi) return; i = uniq[slot]; } else { if (j >= cnt) return; i = slot = i0 + j; }
    const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(key_points + 20 * i);
    uint64_t l[16];
#pragma unroll
    for (int k = 0; k < 8; k++) { ulonglong2 v = src[k]; l[2 * k] = v.x; l[2 * k + 1] = v.y; }     // X, Y, Z (T is not needed)
    fe x, y, z;
    fe_from_limbs51(x, l); fe_from_limbs51(y, l + 5); fe_from_limbs51(z, l + 10);
    uint32_t zw[8];
    fe_tobytes_words(zw, z);
    uint32_t rest = zw[0] ^ 1u;
#pragma unroll
    for (int k = 1; k < 8; k++) rest |= zw[k];
    if (rest) {                                             // Z != 1: affine coordinates need 1 / Z
        fe zi;
        if (F64) fe_invert_f64(zi, z); else fe_invert(zi, z);
        fe_mul(x, x, zi); fe_mul(y, y, zi);
    }
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    ge_niels_packed p; ge_niels_pack(p, nl);
    uint4 *o = reinterpret_cast<uint4 *>(points_A + slot);
#pragma unroll
    for (int k = 0; k < 6; k++) o[k] = make_uint4(p.w[4 * k], p.w[4 * k + 1], p.w[4 * k + 2], p.w[4 * k + 3]);
}

// all keys distinct: scalar of key `pos` is the z h of its only signature
__global__ void k_key_gather(const uint32_t *__restrict__ zh, const uint32_t *__restrict__ uniq, size_t nkeys, uint32_t *__restrict__ out)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nkeys) return;
    const uint4 *src = reinterpret_cast<const uint4 *>(zh + 8 * (size_t)uniq[j]);
    uint4 *dst = reinterpret_cast<uint4 *>(out + 8 * j);
    dst[0] = src[0]; dst[1] = src[1];
}

// acc[dense id][k] += word k of z_i h_i  (64-bit counters: at most 2^31 summands of 32 bits)
__global__ void __launch_bounds__(256)
k_key_accumulate(const uint32_t *__restrict__ zh, const uint32_t *__restrict__ rep, const uint32_t *__restrict__ dense, size_t n,
                 unsigned long long *__restrict__ acc)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long *a = acc + 8 * (size_t)dense[rep[i]];
#pragma unroll
    for (int k = 0; k < 8; k++) atomicAdd(a + k, (unsigned long long)zh[8 * i + k]);
}

// carry the eight counters of a key into one integer S = sum of its c_i = (z_i h_i mod l)  (< 2^287) and reduce it
// modulo 8 l, the exponent of the WHOLE curve group: the reference adds [c_i] A for every signature (batch.rs:240-244),
// and sum [c_i] A = [S] A = [S mod 8l] A also when A carries a small-order component, which a reduction mod l would
// not preserve (l = 5 mod 8).  S mod 8l = 8 ((S >> 3) mod l) + (S & 7) < 2^256.
__global__ void k_key_finalize(const unsigned long long *__restrict__ acc, size_t nkeys, uint32_t *__restrict__ out)
{
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nkeys) return;
    uint32_t x[16];
    unsigned long long carry = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        unsigned long long v = acc[8 * j + k];
        unsigned long long lo = (v & 0xffffffffull) + (carry & 0xffffffffull);
        x[k] = (uint32_t)lo;
        carry = (v >> 32) + (carry >> 32) + (lo >> 32);
    }
    x[8] = (uint32_t)carry; x[9] = (uint32_t)(carry >> 32);
#pragma unroll
    for (int k = 10; k < 16; k++) x[k] = 0;
    const uint32_t low3 = x[0] & 7u;
#pragma unroll
    for (int k = 0; k < 15; k++) x[k] = (x[k] >> 3) | (x[k + 1] << 29);
    x[15] >>= 3;
    uint32_t r[8];
    sc_reduce512(r, x);                                     // < l < 2^253
#pragma unroll
    for (int k = 7; k > 0; k--) r[k] = (r[k] << 3) | (r[k - 1] >> 29);
    r[0] = (r[0] << 3) | low3;
#pragma unroll
    for (int k = 0; k < 8; k++) out[8 * j + k] = r[k];
}

// per batch of `batch` signatures: bit 0 = some s not canonical, bit 1 = some R undecodable, bit 2 = some key undecodable
__global__ void k_batch_status(const uint8_t *__restrict__ bad_s, const uint8_t *__restrict__ bad_r, const uint8_t *__restrict__ bad_key,
                               const uint32_t *__restrict__ rep, const uint32_t *__restrict__ dense, int merged, size_t n, size_t batch,
                               size_t nbatches, uint8_t *__restrict__ out)
{
    size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nbatches) return;
    uint32_t v = 0;
    const size_t hi = min(n, (k + 1) * batch);
    for (size_t i = k * batch; i < hi; i++) {
        const size_t slot = merged ? dense[rep[i]] : i;
        v |= (uint32_t)bad_s[i] | ((uint32_t)bad_r[i] << 1) | ((uint32_t)bad_key[slot] << 2);
    }
    out[k] = (uint8_t)v;
}

// Small-order part of every batch's equation, exactly.  verify_batches tests SUMS of batch equations first (one
// equation over a range of batches, bisected on failure).  Writing E_k = P_k + T_k for the value of batch k's equation
// (batch.rs:240-244; P_k in the prime-order subgroup, T_k in E[8]), a range sum that vanishes settles the P_k -- the
// z_i of different batches come from different transcripts, so a non-zero P_k survives in the sum except with the
// probability a forged signature survives batch.rs itself -- but NOT the T_k: three bits of z_i are all that multiply a
// small-order component, and T_j + T_k = 0 happens for one input in eight (the reference's own VALIDATIONVECTORS hit
// it).  The small-order part only depends on the scalars modulo 8:
//     T_k = small-order part of  S_k = sum_i (z_i mod 8) R_i + sum_i ((z_i h_i mod l) mod 8) A_i,
// (B is torsion-free) and T_k = 0 <=> [l] S_k = identity.  One group of G lanes per batch: every lane keeps two signed
// sums B_1, B_3 (each scalar residue mod 8 written as a + 3 b, a, b in {-1, 0, 1}), S = B_1 + 3 B_3, a shuffle tree over
// the group (k_batch_torsion); then the 252 doublings of [l] on one thread per batch (k_batch_torsion_test).  Four mixed
// additions per signature and one scalar multiplication per BATCH.
// the group order l = 2^252 + 27742317777372353535851937790883648493 (scalar.rs constants::BASEPOINT_ORDER), low 128 bits
__constant__ uint32_t c_l_low[4] = {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu};

__global__ void __launch_bounds__(128)
k_batch_torsion(const uint32_t *__restrict__ zs /* 4 words each */, const uint32_t *__restrict__ zh /* 8 words each: z_i h_i mod l */,
                const ge_niels_packed *__restrict__ pts_R, const ge_niels_packed *__restrict__ pts_A,
                const uint32_t *__restrict__ rep, const uint32_t *__restrict__ dense, int merged, size_t n, size_t batch,
                size_t nbatches, uint32_t G, ge_p3_raw *__restrict__ sums)
{
    const size_t gt = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t k = gt / G;
    const uint32_t gl = (uint32_t)(gt % G);
    const bool live = k < nbatches;                          // dead groups run along with no signatures: the warp stays converged
    const size_t lo = live ? k * batch : 0, hi = live ? min(n, (k + 1) * batch) : 0;
    fe64 d2; fe64_const_2d(d2);
    // every residue k mod 8 is a + 3 b with a, b in {-1, 0, 1}: two signed accumulators, S = B1 + 3 B3, two (uniformly
    // executed) mixed additions per point.  Any integer congruent to the scalar mod 8 gives the same small-order part.
    ge64_p3 B1, B3;
    ge64_identity(B1); ge64_identity(B3);
    const size_t trips = (batch + G - 1) / G;                // the same trip count in every lane
#pragma unroll 1
    for (size_t t = 0; t < trips; t++) {
        const size_t i = lo + t * G + gl;
        const bool have = i < hi;
#pragma unroll 1
        for (int which = 0; which < 2; which++) {
            uint32_t k = 0;
            ge64_niels nl;
            if (have) {
                const ge_niels_packed *src = which == 0 ? pts_R + i : pts_A + (merged ? (size_t)dense[rep[i]] : i);
                k = (which == 0 ? zs[4 * i] : zh[8 * i]) & 7u;
                ge_niels_packed pk;
                const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
#pragma unroll
                for (int q = 0; q < 6; q++) { uint4 v = s4[q]; pk.w[4 * q] = v.x; pk.w[4 * q + 1] = v.y; pk.w[4 * q + 2] = v.z; pk.w[4 * q + 3] = v.w; }
                ge64_niels_unpack(nl, pk);
            }
            //            k:  0  1   2  3  4   5   6   7
            // a (weight 1):  0  1  -1  0  1   0   1  -1          k = a + 3 b (mod 8)
            // b (weight 3):  0  0   1  1  1  -1  -1   0
            const uint32_t a_nz = (0xd6u >> k) & 1u, a_neg = (0x84u >> k) & 1u;
            const uint32_t b_nz = (0x7cu >> k) & 1u, b_neg = (0x60u >> k) & 1u;
            if (a_nz) ge64_madd(B1, B1, nl, a_neg);
            if (b_nz) ge64_madd(B3, B3, nl, b_neg);
        }
    }
    ge64_p3 S, X;
    ge64_dbl(S, B3); ge64_add_p3(S, S, B3, d2); ge64_add_p3(S, S, B1, d2);     // 3 B3 + B1
    for (uint32_t d = G >> 1; d > 0; d >>= 1) { ge64_shfl_down(X, S, (int)d); ge64_add_p3(S, S, X, d2); }
    if (live && gl == 0) {
        ge_p3 q; ge64_to_p3(q, S);
        ge_p3_raw r; ge_p3_store_raw(r, q);
        uint4 *o = reinterpret_cast<uint4 *>(sums + k);
#pragma unroll
        for (int w = 0; w < 10; w++) o[w] = make_uint4(r.w[4 * w], r.w[4 * w + 1], r.w[4 * w + 2], r.w[4 * w + 3]);
    }
}

// [l] S_k == identity ?  One thread per batch (the lanes of k_batch_torsion would all repeat the same 252 doublings):
// left to right over the bits of l below the leading one (bits 251..128 are zero).
__global__ void __launch_bounds__(64)
k_batch_torsion_test(const ge_p3_raw *__restrict__ sums, size_t nbatches, uint8_t *__restrict__ status)
{
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nbatches) return;
    fe64 d2; fe64_const_2d(d2);
    ge_p3 s3;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(sums + k);
        ge_p3_raw r;
#pragma unroll
        for (int w = 0; w < 10; w++) { uint4 v = src[w]; r.w[4 * w] = v.x; r.w[4 * w + 1] = v.y; r.w[4 * w + 2] = v.z; r.w[4 * w + 3] = v.w; }
        ge_p3_load_raw(s3, r);
    }
    ge64_p3 S;
    fe64_from_fe_limbs(S.X, s3.X); fe64_from_fe_limbs(S.Y, s3.Y); fe64_from_fe_limbs(S.Z, s3.Z); fe64_from_fe_limbs(S.T, s3.T);
    ge64_pniels Sn;
    fe64_add(Sn.YpX, S.Y, S.X); fe64_sub(Sn.YmX, S.Y, S.X); Sn.Z = S.Z; fe64_mul(Sn.T2d, S.T, d2);
    fe64_carry(Sn.YpX, Sn.YpX); fe64_carry(Sn.YmX, Sn.YmX);
    ge64_p3 Q = S;
#pragma unroll 1
    for (int b = 251; b >= 0; b--) {
        ge64_dbl(Q, Q);
        if (b < 128 && ((c_l_low[b >> 5] >> (b & 31)) & 1u)) ge64_padd(Q, Q, Sn, 0u);
    }
    ge_p3 q; ge64_to_p3(q, Q);
    if (!ge_is_identity(q)) status[k] |= 8;
}

// signatures of batches that already have a verdict (malformed input or a small-order defect) leave the equations:
// their coefficients become zero, so the range sums of verify_batches_tail only carry the undecided batches
__global__ void k_batch_mask(const uint8_t *__restrict__ status, size_t n, size_t batch, uint32_t *__restrict__ zsprod,
                             uint32_t *__restrict__ zh, uint32_t *__restrict__ z_R)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !status[i / batch]) return;
    const uint4 zero = make_uint4(0, 0, 0, 0);
    uint4 *a = reinterpret_cast<uint4 *>(zsprod + 8 * i), *b = reinterpret_cast<uint4 *>(zh + 8 * i), *c = reinterpret_cast<uint4 *>(z_R + 8 * i);
    a[0] = zero; a[1] = zero; b[0] = zero; b[1] = zero; c[0] = zero; c[1] = zero;
}

// ------------------------------------------------------------------------------------------
// MSM inputs: scalars/points [0] = (-sum z s, B); [1 .. 1+K) = the K distinct keys (K = n without merging);
// [1+n .. 1+2n) = (z_i, R_i).  counters: [0] running number of distinct keys, [1+p] its value after piece p, [15] = 0.
struct VerifyBufs { uint32_t *hrams, *hs, *zsprod, *zs, *scalars; ge_niels_packed *points; int *flags;
                    uint32_t *table, tmask, *rep, *uniq, *dense, *counters; uint8_t *bad_s, *bad_r, *bad_key; };

static int verify_reserve(dalek_b200_ctx *ctx, size_t n, VerifyBufs &b)
{
    int rc;
    const size_t m = 2 * n + 1;
    if (m >= (1ull << 31)) return DALEK_E_INVALID_ARG;
    if ((rc = msm_driver_ws_reserve(ctx))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_HRAM], std::max<size_t>(1, n) * 64))) return rc;   // hrams
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_H], std::max<size_t>(1, n) * 32))) return rc;   // h_i
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_ZS_PROD], std::max<size_t>(1, n) * 32))) return rc;   // z_i s_i
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_Z], std::max<size_t>(1, n) * 16))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_SCALARS], m * 32))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_OUT], m * sizeof(ge_niels_packed)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_SUMS], (size_t)32768 * 9 * 4))) return rc;
    b.hrams = (uint32_t *)ctx->ws[WS_VERIFY_HRAM].p; b.hs = (uint32_t *)ctx->ws[WS_VERIFY_H].p; b.zsprod = (uint32_t *)ctx->ws[WS_VERIFY_ZS_PROD].p;
    b.zs = (uint32_t *)ctx->ws[WS_VERIFY_Z].p; b.scalars = (uint32_t *)ctx->ws[WS_SCALARS].p; b.points = (ge_niels_packed *)ctx->ws[WS_STAGING_OUT].p;
    b.flags = (int *)ctx->ws[WS_FLAGS].p;
    // key de-duplication table: power of two >= 2n slots, plus rep[n], uniq[n], dense[n] and 16 counters
    size_t tsize = 1024;
    while (tsize < 2 * n) tsize <<= 1;
    const size_t n1 = std::max<size_t>(1, n);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_KEY_TABLE], (tsize + 3 * n1 + 16) * 4))) return rc;
    b.table = (uint32_t *)ctx->ws[WS_VERIFY_KEY_TABLE].p; b.tmask = (uint32_t)(tsize - 1);
    b.rep = b.table + tsize; b.uniq = b.rep + n1; b.dense = b.uniq + n1; b.counters = b.dense + n1;
    if (ctx->opt_dedupe_keys) {
        CUDA_TRY(ctx, cudaMemsetAsync(b.table, 0xff, tsize * 4, ctx->stream));
        CUDA_TRY(ctx, cudaMemsetAsync(b.counters, 0, 64, ctx->stream));
    }
    if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_MARKS], 3 * n1))) return rc;          // per-signature / per-key failure marks
    b.bad_s = (uint8_t *)ctx->ws[WS_VERIFY_MARKS].p; b.bad_r = b.bad_s + n1; b.bad_key = b.bad_r + n1;
    CUDA_TRY(ctx, cudaMemsetAsync(b.bad_s, 0, 3 * n1, ctx->stream));
    return 0;
}

// What one verify_batch[es] call adds to the context's options.
struct VerifyCall {
    // signatures per transcript: the batch size of a verify_batches call, else the verify_chunk option.  0 (the
    // default): ONE transcript over the whole batch, the reference's (batch.rs:168-222); it needs every hram first, so
    // it runs in verify_whole_transcript after the last piece.  > 0: one transcript per chunk.
    uint32_t chunk;
    const uint64_t *d_key_points;   // device: the callers' decompressed key points (..._points calls), or null
    size_t batch;                   // 0: one verdict (verify_batch); > 0: independent batches of this many signatures
    int32_t *verdicts;              // one per batch (batch > 0)
};

// Front end for signatures [i0, i1) (i0 a multiple of call.chunk): hashing on stream_hash; transcript and coefficients
// on a high-priority stream (the main one for even pieces, stream3 for odd ones: a transcript kernel is a
// latency-bound chain of Keccak permutations on few warps, so consecutive pieces should overlap);
// decompression on the low-priority stream.  All wait for `ready` if given.
static int verify_front(dalek_b200_ctx *ctx, const VerifyCall &call, const VerifyBufs &b, const uint8_t *d_msgs, const uint64_t *d_offs,
                        const uint32_t *d_sigs, const uint32_t *d_keys, size_t n, size_t i0, size_t i1, cudaEvent_t ready, int piece)
{
    cudaStream_t st = (piece & 1) ? ctx->stream3 : ctx->stream, st2 = ctx->stream2, sh = ctx->stream_hash;
    const size_t cnt = i1 - i0;
    const uint32_t chunk = call.chunk;
    if (ready) { CUDA_TRY(ctx, cudaStreamWaitEvent(sh, ready, 0)); CUDA_TRY(ctx, cudaStreamWaitEvent(st2, ready, 0)); }
    if (cnt) {
        // the hashing -> transcript chain has little parallelism in its second stage: enqueue it first.  SHA-512 of every
        // piece runs on its own stream, so the hashing of piece k+2 is not queued behind the transcripts of piece k
        k_hram<<<cdiv(cnt, 128), 128, 0, sh>>>(d_msgs, d_offs + i0, d_sigs + 16 * i0, d_keys + 8 * i0, cnt, b.hrams + 16 * i0,
                                               b.hs + 8 * i0, b.flags, b.bad_s + i0);
        ctx->launches++;
        trace_mark(ctx, "hram done (hash stream)", sh);
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_hram[piece & 7], sh));
        CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_hram[piece & 7], 0));
        if (chunk) {
            launch_transcripts(ctx, st, b.hrams + 16 * i0, d_sigs + 16 * i0, cnt, chunk, b.zs + 4 * i0);
            trace_mark(ctx, "transcript done (transcript stream)", st);
        }
    }
    ge_niels_packed *points_A = b.points + 1;
    if (piece < 8) { CUDA_TRY(ctx, cudaEventRecord(ctx->ev_prep[piece][0], st2)); ctx->prep_pieces = piece + 1; }
    if (ctx->opt_decompress_f64)
        k_prep_R<1><<<cdiv(cnt + 1, 128), 128, 0, st2>>>(d_sigs + 16 * i0, cnt, b.points + 1 + n + i0, i0 == 0 ? b.points : nullptr, b.flags, b.bad_r + i0);
    else
        k_prep_R<0><<<cdiv(cnt + 1, 128), 128, 0, st2>>>(d_sigs + 16 * i0, cnt, b.points + 1 + n + i0, i0 == 0 ? b.points : nullptr, b.flags, b.bad_r + i0);
    ctx->launches++;
    if (piece < 8) CUDA_TRY(ctx, cudaEventRecord(ctx->ev_prep[piece][1], st2));
    trace_mark(ctx, "prep_R done (decompress stream)", st2);
    if (ctx->opt_dedupe_keys) {
        // keys first seen in this piece are uniq[counters[piece] .. counters[1 + piece])  (counters[15] = 0 for piece 0)
        const uint32_t *lo = piece ? b.counters + piece : b.counters + 15, *hi = b.counters + 1 + piece;
        if (cnt) k_key_dedupe<<<cdiv(cnt, 256), 256, 0, st2>>>(d_keys, i0, cnt, b.table, b.tmask, b.rep, b.uniq, b.dense, b.counters,
                                                               make_uint4(ctx->hash_seed[0], ctx->hash_seed[1], ctx->hash_seed[2], ctx->hash_seed[3]));
        CUDA_TRY(ctx, cudaMemcpyAsync(b.counters + 1 + piece, b.counters, 4, cudaMemcpyDeviceToDevice, st2));
        if (cnt && call.d_key_points) k_prep_A_points<1><<<cdiv(cnt, 128), 128, 0, st2>>>(call.d_key_points, b.uniq, lo, hi, i0, cnt, points_A);
        else if (cnt && ctx->opt_decompress_f64) k_prep_A<1><<<cdiv(cnt, 128), 128, 0, st2>>>(d_keys, b.uniq, lo, hi, i0, cnt, points_A, b.flags, b.bad_key);
        else if (cnt) k_prep_A<0><<<cdiv(cnt, 128), 128, 0, st2>>>(d_keys, b.uniq, lo, hi, i0, cnt, points_A, b.flags, b.bad_key);
        ctx->launches += cnt ? 2 : 0;
    } else if (cnt) {
        if (call.d_key_points) k_prep_A_points<1><<<cdiv(cnt, 128), 128, 0, st2>>>(call.d_key_points, nullptr, nullptr, nullptr, i0, cnt, points_A);
        else if (ctx->opt_decompress_f64) k_prep_A<1><<<cdiv(cnt, 128), 128, 0, st2>>>(d_keys, nullptr, nullptr, nullptr, i0, cnt, points_A, b.flags, b.bad_key);
        else k_prep_A<0><<<cdiv(cnt, 128), 128, 0, st2>>>(d_keys, nullptr, nullptr, nullptr, i0, cnt, points_A, b.flags, b.bad_key);
        ctx->launches++;
    }
    if (cnt && chunk) {
        // with key merging z_i h_i replaces h_i in place and is summed per key in verify_tail
        uint32_t *out_zh = ctx->opt_dedupe_keys ? b.hs + 8 * i0 : b.scalars + 8 * (1 + i0);
        k_coeffs<<<cdiv(cnt, 128), 128, 0, st>>>(b.zs + 4 * i0, d_sigs + 16 * i0, b.hs + 8 * i0, cnt, b.scalars + 8 * (1 + n + i0),
                                                 out_zh, b.zsprod + 8 * i0);
        ctx->launches++;
        trace_mark(ctx, "coeffs done (transcript stream)", st);
    }
    trace_mark(ctx, "keys done (decompress stream)", st2);
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

// call.chunk = 0: the reference's single transcript over all n signatures (batch.rs:168-222) -- a strictly
// sequential sponge (1.73 Keccak permutations per signature), one warp -- then the coefficients.  Runs on the main
// stream after the hashing of every piece.
static int verify_whole_transcript(dalek_b200_ctx *ctx, const VerifyCall &call, const VerifyBufs &b, const uint32_t *d_sigs, size_t n)
{
    if (call.chunk || !n) return 0;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join2, ctx->stream_hash));       // every piece is hashed on stream_hash
    CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join2, 0));
    launch_transcripts(ctx, st, b.hrams, d_sigs, n, (uint32_t)std::min<size_t>(n, 0xffffffffu), b.zs);
    trace_mark(ctx, "whole-batch transcript done (hash stream)", st);
    uint32_t *out_zh = ctx->opt_dedupe_keys ? b.hs : b.scalars + 8;
    k_coeffs<<<cdiv(n, 128), 128, 0, st>>>(b.zs, d_sigs, b.hs, n, b.scalars + 8 * (1 + n), out_zh, b.zsprod);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

// Joins the two front-end streams and returns the number of distinct keys (n without key merging).
static int verify_join(dalek_b200_ctx *ctx, const VerifyBufs &b, size_t n, int pieces, size_t *nkeys)
{
    int rc;
    cudaStream_t st = ctx->stream, st2 = ctx->stream2;
    ctx->last_zs_n = n;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, st2));
    CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join, 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join2, ctx->stream3));
    CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join2, 0));
    if ((rc = pinned_reserve(ctx, sizeof(MsmResult) + 128))) return rc;
    *nkeys = n;
    trace_mark(ctx, "front end joined", st);
    if (ctx->opt_dedupe_keys && n) {
        // the number of distinct keys sizes the MSM: one small read-back in the middle of the call
        uint32_t *hk = (uint32_t *)((char *)ctx->h_pinned + sizeof(MsmResult) + 64);
        CUDA_TRY(ctx, cudaMemcpyAsync(hk, b.counters + pieces, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
        *nkeys = *hk;
        if (*nkeys == 0 || *nkeys > n) { ctx->last_error = "key table corrupted"; return -4; }
    }
    return 0;
}

// The equation of batch.rs:240-250 restricted to signatures [lo, hi):
//   [-sum z_i s_i] B + sum z_i R_i + sum_keys [sum_{i of that key} z_i h_i] A_key  ==  identity ?
static int verify_equation(dalek_b200_ctx *ctx, const VerifyBufs &b, size_t n, size_t nkeys, size_t lo, size_t hi, bool *is_identity)
{
    int rc;
    cudaStream_t st = ctx->stream;
    const size_t cnt = hi - lo;
    const uint32_t nsum = (uint32_t)std::min<size_t>(32768, std::max<size_t>(1, cnt));
    k_sum_partial<<<cdiv(nsum, 128), 128, 0, st>>>(b.zsprod + 8 * lo, cnt, nsum, (uint32_t *)ctx->ws[WS_VERIFY_SUMS].p);
    k_sum_final<<<1, 256, 0, st>>>((const uint32_t *)ctx->ws[WS_VERIFY_SUMS].p, nsum, b.scalars);
    ctx->launches += 2;
    const bool merged = ctx->opt_dedupe_keys && n;
    if (merged) {
        if (nkeys == n && cnt == n) {
            k_key_gather<<<cdiv(n, 256), 256, 0, st>>>(b.hs, b.uniq, n, b.scalars + 8);
            ctx->launches++;
        } else {
            if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_KEY_ACC], nkeys * 64))) return rc;
            unsigned long long *acc = (unsigned long long *)ctx->ws[WS_VERIFY_KEY_ACC].p;
            CUDA_TRY(ctx, cudaMemsetAsync(acc, 0, nkeys * 64, st));
            if (cnt) k_key_accumulate<<<cdiv(cnt, 256), 256, 0, st>>>(b.hs + 8 * lo, b.rep + lo, b.dense, cnt, acc);
            k_key_finalize<<<cdiv(nkeys, 128), 128, 0, st>>>(acc, nkeys, b.scalars + 8);
            ctx->launches += 2;
        }
    }
    trace_mark(ctx, "sums and per-key scalars done", st);
    // the z_i are 128-bit (batch.rs:224-229): their terms only populate the low windows
    const size_t nlong = merged ? nkeys + 1 : cnt + 1;
    const int c = msm_choose_window_bits_mixed(ctx, cnt, 128, nlong);
    if (merged || cnt == n) {
        if ((rc = msm_accumulate_chunk(ctx, b.scalars, b.points, nlong, c, true))) return rc;
    } else {           // one term per signature, sub-range: the basepoint term, then the keys of the range
        if ((rc = msm_accumulate_chunk(ctx, b.scalars, b.points, 1, c, true))) return rc;
        if (cnt && (rc = msm_accumulate_chunk(ctx, b.scalars + 8 * (1 + lo), b.points + 1 + lo, cnt, c, false))) return rc;
    }
    trace_mark(ctx, "key chunk accumulated", st);
    if (cnt && (rc = msm_accumulate_chunk(ctx, b.scalars + 8 * (1 + n + lo), b.points + 1 + n + lo, cnt, c, false, (128 + c) / c))) return rc;
    trace_mark(ctx, "R chunk accumulated", st);
    if ((rc = msm_reduce_finish(ctx, c, (ge_p3_raw *)ctx->ws[WS_MSM_WINDOWS].p, (MsmResult *)ctx->ws[WS_MSM_RESULT].p))) return rc;
    trace_mark(ctx, "reduced and combined", st);
    MsmResult *h = (MsmResult *)ctx->h_pinned;
    CUDA_TRY(ctx, cudaMemcpyAsync(h, ctx->ws[WS_MSM_RESULT].p, sizeof(MsmResult), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    *is_identity = h->is_identity != 0;
    return 0;
}

// Stage timings of a call: kernel_ms, the bucket kernel of its (first) equation, if it was measured; the R decompression
// of every piece.
static void verify_stage_times(dalek_b200_ctx *ctx, float kernel_ms)
{
    float ms = 0.f;
    if (kernel_ms >= 0.f) ctx->last_kernel_ms = kernel_ms;
    ctx->last_prep_ms = 0.f;
    for (int k = 0; k < ctx->prep_pieces; k++)
        if ((ms = elapsed_ms(ctx->ev_prep[k][0], ctx->ev_prep[k][1])) >= 0.f) ctx->last_prep_ms += ms;
    trace_dump(ctx);
}

// the single verdict of verify_batch
static int verify_tail(dalek_b200_ctx *ctx, const VerifyBufs &b, size_t n, int pieces)
{
    int rc;
    size_t nkeys = 0;
    bool ident = false;
    if ((rc = verify_join(ctx, b, n, pieces, &nkeys))) return rc;
    if ((rc = verify_equation(ctx, b, n, nkeys, 0, n, &ident))) return rc;
    int *hflags = (int *)((char *)ctx->h_pinned + sizeof(MsmResult));
    CUDA_TRY(ctx, cudaMemcpyAsync(hflags, b.flags, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    verify_stage_times(ctx, elapsed_ms(ctx->ev_a, ctx->ev_b));
    // error precedence follows the reference: VerifyingKey::from_bytes happens before verify_batch
    // can be called (PointDecompression); then s canonicity (batch.rs:208-211); then R / equation.
    if (hflags[FLAG_BAD_A]) return ED25519_ERR_POINT_DECOMPRESSION;
    if (hflags[FLAG_BAD_S]) return ED25519_ERR_SCALAR_FORMAT;
    if (hflags[FLAG_BAD_R]) return ED25519_ERR_VERIFY;
    return ident ? DALEK_OK : ED25519_ERR_VERIFY;
}

// Many independent batches of `batch` signatures in one call (the result of verify_batch on each).  A batch fails iff
// the value E_k of its equation is not the identity.  Its small-order part is tested exactly for every batch
// (k_batch_torsion); batches that fail there, or carry malformed input, get their verdict and leave the equations
// (k_batch_mask).  For the rest only the prime-order parts are open: the combined equation over all of them is tested
// first -- every batch has its own transcript, so a non-zero prime-order part survives in a sum of batch equations
// except with the probability a forgery survives batch.rs itself -- and only when it fails are halves re-tested down
// to single batches.
static int verify_batches_tail(dalek_b200_ctx *ctx, const VerifyCall &call, const VerifyBufs &b, size_t n, int pieces)
{
    int rc;
    const size_t batch = call.batch;
    size_t nkeys = 0;
    const size_t nb = (n + batch - 1) / batch;
    if ((rc = verify_join(ctx, b, n, pieces, &nkeys))) return rc;
    if (nb == 0) return DALEK_OK;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_ITEM_STATUS], nb))) return rc;
    const int merged = ctx->opt_dedupe_keys ? 1 : 0;
    uint32_t *zh = merged ? b.hs : b.scalars + 8;            // where k_coeffs left z_i h_i
    // The per-batch status (malformed input, small-order defect) is computed on the decompression stream, idle by now, WHILE
    // the main stream evaluates the combined equation over everything.  If that equation holds, every prime-order part is
    // settled and the verdicts follow from the status alone -- the common case costs no serial time for the status kernels
    // (the [l] S_k chains are latency-bound and hide under the bucket kernel).  If it fails, the batches that already have a
    // verdict are masked out of the coefficients and the ranges are examined as before.
    cudaStream_t ss = ctx->stream2;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ss, ctx->ev_fork, 0));
    k_batch_status<<<cdiv(nb, 128), 128, 0, ss>>>(b.bad_s, b.bad_r, b.bad_key, b.rep, b.dense, merged, n, batch, nb, (uint8_t *)ctx->ws[WS_ITEM_STATUS].p);
    {   // lanes per batch: enough groups to fill the machine, at least ~8 signatures per lane
        uint32_t G = 1;
        while (G < 32 && (size_t)G * 8 <= batch && nb * G < (size_t)ctx->sm_count * 512) G <<= 1;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_BATCH_TORSION], nb * sizeof(ge_p3_raw)))) return rc;
        k_batch_torsion<<<cdiv(nb * G, 128), 128, 0, ss>>>(b.zs, zh, b.points + 1 + n, b.points + 1, b.rep, b.dense, merged, n, batch,
                                                           nb, G, (ge_p3_raw *)ctx->ws[WS_BATCH_TORSION].p);
        k_batch_torsion_test<<<cdiv(nb, 64), 64, 0, ss>>>((const ge_p3_raw *)ctx->ws[WS_BATCH_TORSION].p, nb, (uint8_t *)ctx->ws[WS_ITEM_STATUS].p);
    }
    ctx->launches += 3;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ss));
    trace_mark(ctx, "batch status and small-order parts done (decompress stream)", ss);
    bool all_ok = false;
    if ((rc = verify_equation(ctx, b, n, nkeys, 0, n, &all_ok))) return rc;
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    std::vector<uint8_t> status(nb);                                     // (a pageable read-back blocks the host: only now)
    CUDA_TRY(ctx, cudaMemcpyAsync(status.data(), ctx->ws[WS_ITEM_STATUS].p, nb, cudaMemcpyDeviceToHost, ss));
    CUDA_TRY(ctx, cudaStreamSynchronize(ss));
    float first_kernel_ms = elapsed_ms(ctx->ev_a, ctx->ev_b);
    std::vector<uint8_t> eq_ok(nb, 0);
    // ranges of batches still to be classified; `known_bad`: the range is known to contain a failing batch (its parent
    // failed and its sibling verified), so its own equation need not be evaluated again
    struct Range { size_t k0, k1; bool known_bad; };
    std::vector<Range> todo;
    if (all_ok) {
        std::fill(eq_ok.begin(), eq_ok.end(), (uint8_t)1);
    } else {
        k_batch_mask<<<cdiv(n, 256), 256, 0, ctx->stream>>>((const uint8_t *)ctx->ws[WS_ITEM_STATUS].p, n, batch, b.zsprod, zh, b.scalars + 8 * (1 + n));
        ctx->launches++;
        todo.push_back({0, nb, false});
    }
    while (!todo.empty()) {
        const Range r = todo.back();
        todo.pop_back();
        bool ident = false;
        if (!r.known_bad) {
            if ((rc = verify_equation(ctx, b, n, nkeys, r.k0 * batch, std::min(n, r.k1 * batch), &ident))) return rc;
            if (ident) { for (size_t k = r.k0; k < r.k1; k++) eq_ok[k] = 1; continue; }
        }
        if (r.k1 - r.k0 == 1) continue;                                  // a single failing batch
        const size_t mid = r.k0 + (r.k1 - r.k0) / 2;
        // left half first; if it verifies, the right half is the failing one
        bool left_ok = false;
        if ((rc = verify_equation(ctx, b, n, nkeys, r.k0 * batch, std::min(n, mid * batch), &left_ok))) return rc;
        if (left_ok) {
            for (size_t k = r.k0; k < mid; k++) eq_ok[k] = 1;
            todo.push_back({mid, r.k1, true});
        } else {
            todo.push_back({mid, r.k1, false});
            todo.push_back({r.k0, mid, true});
        }
    }
    verify_stage_times(ctx, first_kernel_ms);
    int any = 0;
    for (size_t k = 0; k < nb; k++) {
        int v = (status[k] & 4) ? ED25519_ERR_POINT_DECOMPRESSION : (status[k] & 1) ? ED25519_ERR_SCALAR_FORMAT
                : ((status[k] & (2 | 8)) || !eq_ok[k]) ? ED25519_ERR_VERIFY : DALEK_OK;
        call.verdicts[k] = v;
        any |= v;
    }
    return any ? ED25519_ERR_VERIFY : DALEK_OK;
}

// Front end shared with the per-signature verifier (single.cu): SHA-512(R || A || M) mod l (with ph_dom: SHA-512(dom2 ||
// R || A || PH), d_msgs then holding n 64-byte prehashes and d_offs unused) and the canonical-s marks of every signature, public keys de-duplicated (rep / dense / uniq as in verify_batch).  Synchronises to return the number
// of distinct keys.  The arrays stay in their roles (WS_VERIFY_H, WS_VERIFY_MARKS, WS_VERIFY_KEY_TABLE) until the caller's
// public call returns: nothing the caller runs after this function reserves them.
int verify_each_front(dalek_b200_ctx *ctx, const uint8_t *d_msgs, const uint64_t *d_offs, const uint32_t *d_sigs, const uint32_t *d_keys,
                      size_t n, EachFront *out, const Sha512Prefix *ph_dom)
{
    int rc;
    VerifyBufs b;
    if ((rc = verify_reserve(ctx, n, b))) return rc;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaMemsetAsync(b.flags, 0, FLAG_WORDS * sizeof(int), st));
    if (!ctx->opt_dedupe_keys) {                       // (verify_reserve only clears the table when merging is on)
        CUDA_TRY(ctx, cudaMemsetAsync(b.table, 0xff, ((size_t)b.tmask + 1) * 4, st));
        CUDA_TRY(ctx, cudaMemsetAsync(b.counters, 0, 64, st));
    }
    if (ph_dom) k_hram_ph<<<cdiv(n, 128), 128, 0, st>>>(d_msgs, *ph_dom, d_sigs, d_keys, n, b.hrams, b.hs, b.flags, b.bad_s);
    else k_hram<<<cdiv(n, 128), 128, 0, st>>>(d_msgs, d_offs, d_sigs, d_keys, n, b.hrams, b.hs, b.flags, b.bad_s);
    k_key_dedupe<<<cdiv(n, 256), 256, 0, st>>>(d_keys, 0, n, b.table, b.tmask, b.rep, b.uniq, b.dense, b.counters,
                                               make_uint4(ctx->hash_seed[0], ctx->hash_seed[1], ctx->hash_seed[2], ctx->hash_seed[3]));
    ctx->launches += 2;
    if ((rc = pinned_reserve(ctx, 256))) return rc;
    uint32_t *hk = (uint32_t *)ctx->h_pinned;
    CUDA_TRY(ctx, cudaMemcpyAsync(hk, b.counters, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    out->hs = b.hs; out->bad_s = b.bad_s; out->rep = b.rep; out->dense = b.dense; out->uniq = b.uniq; out->nkeys = *hk;
    if (out->nkeys == 0 || out->nkeys > n) { ctx->last_error = "key table corrupted"; return -4; }
    return 0;
}

// Kinds of verify_batch[es] entry point: where the inputs live, whether the caller passes the decompressed key points,
// whether the call returns one verdict per batch.
enum { VERIFY_DEVICE = 1, VERIFY_POINTS = 2, VERIFY_BATCHES = 4 };

// The arguments of one call: n messages back to back with n + 1 offsets, n signatures (R || s), n keys and, with
// VERIFY_POINTS, the decompressed point of every key (20 u64 limbs each); all in host memory or all in device memory.
struct VerifyArgs { const void *msgs, *offs, *sigs, *keys, *key_points; size_t n, batch; int32_t *verdicts; };

// Every verify_batch[es] entry point: the argument check, then the device inputs read in place or the host inputs
// streamed in up to 8 pieces, then the whole-batch transcript and the tail of the call.
static int verify_call(dalek_b200_ctx *ctx, int kind, const VerifyArgs &a)
{
    const bool on_device = kind & VERIFY_DEVICE, batches = kind & VERIFY_BATCHES;
    const size_t n = a.n;
    const uint8_t *msgs = (const uint8_t *)a.msgs;
    const uint64_t *offs = (const uint64_t *)a.offs;
    if (!ctx || (batches && (!a.batch || a.batch > (1u << 20)))) return DALEK_E_INVALID_ARG;
    if (n && (!a.sigs || !a.keys || ((kind & VERIFY_POINTS) && !a.key_points) || (batches && !a.verdicts))) return DALEK_E_INVALID_ARG;
    if (on_device ? n && !offs : !flat_messages_ok(msgs, offs, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    // every batch of a verify_batches call gets exactly the reference's transcript
    VerifyCall call{(uint32_t)(a.batch ? a.batch : (size_t)ctx->opt_verify_chunk), on_device ? (const uint64_t *)a.key_points : nullptr,
                    a.batch, a.verdicts};
    int rc, pieces = 1;
    VerifyBufs b;
    const uint32_t *d_sigs = (const uint32_t *)a.sigs;
    if (on_device) {
        if ((rc = verify_reserve(ctx, n, b))) return rc;
        CUDA_TRY(ctx, cudaMemsetAsync(b.flags, 0, FLAG_WORDS * sizeof(int), ctx->stream));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
        if ((rc = verify_front(ctx, call, b, msgs, offs, d_sigs, (const uint32_t *)a.keys, n, 0, n, ctx->ev_fork, 0))) return rc;
    } else {
        const uint8_t *sigs = (const uint8_t *)a.sigs, *pubkeys = (const uint8_t *)a.keys;
        const uint64_t *key_points = (const uint64_t *)a.key_points;
        size_t mbytes = n ? (size_t)offs[n] : 0;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], mbytes + 16))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_MSG_OFFSETS], (n + 1) * 8))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], std::max<size_t>(1, n) * 96))) return rc;   // sigs + keys
        if ((rc = verify_reserve(ctx, n, b))) return rc;
        uint8_t *d_msgs = (uint8_t *)ctx->ws[WS_STAGING_MSGS].p, *d_sig8 = (uint8_t *)ctx->ws[WS_STAGING_IN].p, *d_keys = d_sig8 + n * 64;
        if (key_points) {
            if ((rc = ws_reserve(ctx, ctx->ws[WS_VERIFY_KEY_POINTS], std::max<size_t>(1, n) * 160))) return rc;
            call.d_key_points = (const uint64_t *)ctx->ws[WS_VERIFY_KEY_POINTS].p;
        }
        uint64_t *d_offs = (uint64_t *)ctx->ws[WS_MSG_OFFSETS].p;
        d_sigs = (const uint32_t *)d_sig8;
        cudaStream_t st = ctx->stream, sc = ctx->stream_copy;
        CUDA_TRY(ctx, cudaMemsetAsync(b.flags, 0, FLAG_WORDS * sizeof(int), st));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
        CUDA_TRY(ctx, cudaStreamWaitEvent(sc, ctx->ev_fork, 0));
        // stream the batch in up to 8 pieces (boundaries on call.chunk multiples): the copy of piece k+1
        // overlaps hashing / decompression of piece k
        const size_t vc = std::max<size_t>(1, call.chunk);
        pieces = n >= (1u << 18) ? (int)std::min<long>(8, std::max<long>(1, ctx->opt_verify_pieces)) : 1;
        size_t prev = 0;
        for (int k = 0; k < pieces; k++) {
            size_t i1 = k == pieces - 1 ? n : std::min(n, ((n * (k + 1) / pieces) / vc) * vc);     // equal pieces: the front end outlasts the copies
            size_t i0 = prev, cnt = i1 - i0;
            prev = i1;
            if (cnt) {
                size_t m0 = (size_t)offs[i0], m1 = (size_t)offs[i1];
                if (m1 > m0) CUDA_TRY(ctx, cudaMemcpyAsync(d_msgs + m0, msgs + m0, m1 - m0, cudaMemcpyHostToDevice, sc));
                CUDA_TRY(ctx, cudaMemcpyAsync(d_offs + i0, offs + i0, (cnt + 1) * 8, cudaMemcpyHostToDevice, sc));
                CUDA_TRY(ctx, cudaMemcpyAsync(d_sig8 + i0 * 64, sigs + i0 * 64, cnt * 64, cudaMemcpyHostToDevice, sc));
                CUDA_TRY(ctx, cudaMemcpyAsync(d_keys + i0 * 32, pubkeys + i0 * 32, cnt * 32, cudaMemcpyHostToDevice, sc));
                if (key_points) CUDA_TRY(ctx, cudaMemcpyAsync((char *)ctx->ws[WS_VERIFY_KEY_POINTS].p + i0 * 160, key_points + 20 * i0, cnt * 160, cudaMemcpyHostToDevice, sc));
            }
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_grp[k], sc));
            if ((rc = verify_front(ctx, call, b, d_msgs, d_offs, d_sigs, (const uint32_t *)d_keys, n, i0, i1, ctx->ev_grp[k], k))) return rc;
        }
    }
    if ((rc = verify_whole_transcript(ctx, call, b, d_sigs, n))) return rc;
    return call.batch ? verify_batches_tail(ctx, call, b, n, pieces) : verify_tail(ctx, b, n, pieces);
}

extern "C" {

int ed25519_b200_verify_batch_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                       const void *d_sigs, const void *d_pubkeys, size_t n, size_t msgs_bytes)
{
    (void)msgs_bytes;
    return verify_call(ctx, VERIFY_DEVICE, {d_msgs_flat, d_msg_offsets, d_sigs, d_pubkeys, nullptr, n, 0, nullptr});
}

int ed25519_b200_verify_batch_flat_points_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                              const void *d_sigs, const void *d_pubkeys, const void *d_key_points, size_t n)
{
    return verify_call(ctx, VERIFY_DEVICE | VERIFY_POINTS, {d_msgs_flat, d_msg_offsets, d_sigs, d_pubkeys, d_key_points, n, 0, nullptr});
}

int ed25519_b200_verify_batch_flat_points(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                          const uint8_t *sigs, const uint8_t *pubkeys, const uint64_t *key_points, size_t n)
{
    return verify_call(ctx, VERIFY_POINTS, {msgs_flat, msg_offsets, sigs, pubkeys, key_points, n, 0, nullptr});
}

int ed25519_b200_verify_batches_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets,
                                         const void *d_sigs, const void *d_pubkeys, size_t n, size_t batch_size, int32_t *verdicts)
{
    return verify_call(ctx, VERIFY_DEVICE | VERIFY_BATCHES, {d_msgs_flat, d_msg_offsets, d_sigs, d_pubkeys, nullptr, n, batch_size, verdicts});
}

int ed25519_b200_verify_batches_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                     const uint8_t *sigs, const uint8_t *pubkeys, size_t n, size_t batch_size, int32_t *verdicts)
{
    return verify_call(ctx, VERIFY_BATCHES, {msgs_flat, msg_offsets, sigs, pubkeys, nullptr, n, batch_size, verdicts});
}

int ed25519_b200_verify_batches_flat_points_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets, const void *d_sigs,
                                                const void *d_pubkeys, const void *d_key_points, size_t n, size_t batch_size, int32_t *verdicts)
{
    return verify_call(ctx, VERIFY_DEVICE | VERIFY_POINTS | VERIFY_BATCHES,
                       {d_msgs_flat, d_msg_offsets, d_sigs, d_pubkeys, d_key_points, n, batch_size, verdicts});
}

int ed25519_b200_verify_batches_flat_points(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, const uint8_t *sigs,
                                            const uint8_t *pubkeys, const uint64_t *key_points, size_t n, size_t batch_size, int32_t *verdicts)
{
    return verify_call(ctx, VERIFY_POINTS | VERIFY_BATCHES, {msgs_flat, msg_offsets, sigs, pubkeys, key_points, n, batch_size, verdicts});
}

int ed25519_b200_verify_batch_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets,
                                   const uint8_t *sigs, const uint8_t *pubkeys, size_t n)
{
    return verify_call(ctx, 0, {msgs_flat, msg_offsets, sigs, pubkeys, nullptr, n, 0, nullptr});
}

int ed25519_b200_verify_batch(dalek_b200_ctx *ctx, const uint8_t *const *msgs, const size_t *msg_lens,
                              const uint8_t *sigs, const uint8_t *pubkeys, size_t n)
{
    if (n && (!msgs || !msg_lens)) return DALEK_E_INVALID_ARG;             // the gather reads these; verify_call checks the rest
    // gather the messages into one staging buffer (multi-threaded for large batches)
    std::vector<uint64_t> offs(n + 1);
    offs[0] = 0;
    for (size_t i = 0; i < n; i++) offs[i + 1] = offs[i] + msg_lens[i];
    std::vector<uint8_t> flat(offs[n] + 1);
    unsigned nt = n > (1u << 16) ? std::min(16u, std::max(1u, std::thread::hardware_concurrency())) : 1;
    auto work = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; i++) if (msg_lens[i]) memcpy(flat.data() + offs[i], msgs[i], msg_lens[i]);
    };
    if (nt <= 1) work(0, n);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; t++) th.emplace_back(work, n * t / nt, n * (t + 1) / nt);
        for (auto &x : th) x.join();
    }
    return ed25519_b200_verify_batch_flat(ctx, flat.data(), offs.data(), sigs, pubkeys, n);
}

int ed25519_b200_last_zs(dalek_b200_ctx *ctx, uint8_t *zs_out, size_t n)
{
    if (!ctx || !zs_out || n > ctx->last_zs_n) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (n) CUDA_TRY(ctx, cudaMemcpy(zs_out, ctx->ws[WS_VERIFY_Z].p, n * 16, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
