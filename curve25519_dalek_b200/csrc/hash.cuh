// hash.cuh -- device SHA-512 (FIPS 180-4) and the STROBE-128 / Merlin subset that
// ed25519-dalek's verify_batch draws its coefficients from (ed25519-dalek/src/batch.rs:168-222,
// src/batch/transcript.rs:39-207; third-party sha2 0.11 / strobe-rs 0.13 / keccak 0.2).
// One thread runs one hash / one sponge; state lives in registers / local memory.
#pragma once
#include <stdint.h>

// ---------------------------------------------------------------- SHA-512
static __device__ __constant__ uint64_t SHA512_K[80] = {
    0x428a2f98d728ae22ULL, 0x7137449123ef65cdULL, 0xb5c0fbcfec4d3b2fULL, 0xe9b5dba58189dbbcULL,
    0x3956c25bf348b538ULL, 0x59f111f1b605d019ULL, 0x923f82a4af194f9bULL, 0xab1c5ed5da6d8118ULL,
    0xd807aa98a3030242ULL, 0x12835b0145706fbeULL, 0x243185be4ee4b28cULL, 0x550c7dc3d5ffb4e2ULL,
    0x72be5d74f27b896fULL, 0x80deb1fe3b1696b1ULL, 0x9bdc06a725c71235ULL, 0xc19bf174cf692694ULL,
    0xe49b69c19ef14ad2ULL, 0xefbe4786384f25e3ULL, 0x0fc19dc68b8cd5b5ULL, 0x240ca1cc77ac9c65ULL,
    0x2de92c6f592b0275ULL, 0x4a7484aa6ea6e483ULL, 0x5cb0a9dcbd41fbd4ULL, 0x76f988da831153b5ULL,
    0x983e5152ee66dfabULL, 0xa831c66d2db43210ULL, 0xb00327c898fb213fULL, 0xbf597fc7beef0ee4ULL,
    0xc6e00bf33da88fc2ULL, 0xd5a79147930aa725ULL, 0x06ca6351e003826fULL, 0x142929670a0e6e70ULL,
    0x27b70a8546d22ffcULL, 0x2e1b21385c26c926ULL, 0x4d2c6dfc5ac42aedULL, 0x53380d139d95b3dfULL,
    0x650a73548baf63deULL, 0x766a0abb3c77b2a8ULL, 0x81c2c92e47edaee6ULL, 0x92722c851482353bULL,
    0xa2bfe8a14cf10364ULL, 0xa81a664bbc423001ULL, 0xc24b8b70d0f89791ULL, 0xc76c51a30654be30ULL,
    0xd192e819d6ef5218ULL, 0xd69906245565a910ULL, 0xf40e35855771202aULL, 0x106aa07032bbd1b8ULL,
    0x19a4c116b8d2d0c8ULL, 0x1e376c085141ab53ULL, 0x2748774cdf8eeb99ULL, 0x34b0bcb5e19b48a8ULL,
    0x391c0cb3c5c95a63ULL, 0x4ed8aa4ae3418acbULL, 0x5b9cca4f7763e373ULL, 0x682e6ff3d6b2b8a3ULL,
    0x748f82ee5defb2fcULL, 0x78a5636f43172f60ULL, 0x84c87814a1f0ab72ULL, 0x8cc702081a6439ecULL,
    0x90befffa23631e28ULL, 0xa4506cebde82bde9ULL, 0xbef9a3f7b2c67915ULL, 0xc67178f2e372532bULL,
    0xca273eceea26619cULL, 0xd186b8c721c0c207ULL, 0xeada7dd6cde0eb1eULL, 0xf57d4f7fee6ed178ULL,
    0x06f067aa72176fbaULL, 0x0a637dc5a2c898a6ULL, 0x113f9804bef90daeULL, 0x1b710b35131c471bULL,
    0x28db77f523047d84ULL, 0x32caab7b40c72493ULL, 0x3c9ebe0a15c9bebcULL, 0x431d67c49c100d4cULL,
    0x4cc5d4becb3e42b6ULL, 0x597f299cfc657e2aULL, 0x5fcb6fab3ad6faecULL, 0x6c44198c4a475817ULL};

__device__ __forceinline__ uint64_t ror64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

struct sha512_state {
    uint64_t h[8];
    uint64_t w[16];     // current block, big-endian words being filled
    uint32_t fill;      // bytes in the current block
    uint64_t total;     // total bytes absorbed
};

__device__ __forceinline__ void sha512_init(sha512_state &s)
{
    s.h[0] = 0x6a09e667f3bcc908ULL; s.h[1] = 0xbb67ae8584caa73bULL; s.h[2] = 0x3c6ef372fe94f82bULL;
    s.h[3] = 0xa54ff53a5f1d36f1ULL; s.h[4] = 0x510e527fade682d1ULL; s.h[5] = 0x9b05688c2b3e6c1fULL;
    s.h[6] = 0x1f83d9abfb41bd6bULL; s.h[7] = 0x5be0cd19137e2179ULL;
#pragma unroll
    for (int i = 0; i < 16; i++) s.w[i] = 0;
    s.fill = 0; s.total = 0;
}

static __device__ __noinline__ void sha512_compress(uint64_t h[8], uint64_t w[16])
{
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
    for (int r = 0; r < 80; r += 16) {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (r) {
                uint64_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
                uint64_t s0 = ror64(w15, 1) ^ ror64(w15, 8) ^ (w15 >> 7);
                uint64_t s1 = ror64(w2, 19) ^ ror64(w2, 61) ^ (w2 >> 6);
                w[i] = w[i] + s0 + w[(i + 9) & 15] + s1;
            }
            uint64_t S1 = ror64(e, 14) ^ ror64(e, 18) ^ ror64(e, 41);
            uint64_t ch = (e & f) ^ (~e & g);
            uint64_t t1 = hh + S1 + ch + SHA512_K[r + i] + w[i];
            uint64_t S0 = ror64(a, 28) ^ ror64(a, 34) ^ ror64(a, 39);
            uint64_t mj = (a & b) ^ (a & c) ^ (b & c);
            uint64_t t2 = S0 + mj;
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

__device__ __forceinline__ void sha512_put_byte(sha512_state &s, uint32_t byte)
{
    uint32_t wi = s.fill >> 3, sh = 56 - 8 * (s.fill & 7);
    s.w[wi] |= (uint64_t)byte << sh;
    if (++s.fill == 128) {
        sha512_compress(s.h, s.w);
#pragma unroll
        for (int i = 0; i < 16; i++) s.w[i] = 0;
        s.fill = 0;
    }
}

__device__ __forceinline__ void sha512_update(sha512_state &s, const uint8_t *p, size_t len)
{
    s.total += len;
    for (size_t i = 0; i < len; i++) sha512_put_byte(s, p[i]);
}

// absorb 8 little-endian 32-bit words (a 32-byte string held in registers)
__device__ __forceinline__ void sha512_update_words(sha512_state &s, const uint32_t w[8])
{
    s.total += 32;
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int b = 0; b < 4; b++) sha512_put_byte(s, (w[i] >> (8 * b)) & 0xff);
}

// digest as 16 little-endian 32-bit words (= the 64 output bytes read as LE words)
__device__ __forceinline__ void sha512_final_words(sha512_state &s, uint32_t out[16])
{
    uint64_t bits = s.total * 8;
    sha512_put_byte(s, 0x80);
    while (s.fill != 112) sha512_put_byte(s, 0);
    s.w[14] = 0; s.w[15] = bits;
    sha512_compress(s.h, s.w);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint64_t v = s.h[i];                   // big-endian 8 bytes -> two LE words
        out[2 * i] = __byte_perm((uint32_t)(v >> 32), 0, 0x0123);
        out[2 * i + 1] = __byte_perm((uint32_t)v, 0, 0x0123);
    }
}

// One SHA-512 compression with the block in registers (static word indices, no staging buffer in local memory).
__device__ __forceinline__ void sha512_compress_regs(uint64_t h[8], uint64_t w[16])
{
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
    for (int r = 0; r < 80; r += 16) {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (r) {
                uint64_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
                uint64_t s0 = ror64(w15, 1) ^ ror64(w15, 8) ^ (w15 >> 7);
                uint64_t s1 = ror64(w2, 19) ^ ror64(w2, 61) ^ (w2 >> 6);
                w[i] = w[i] + s0 + w[(i + 9) & 15] + s1;
            }
            uint64_t S1 = ror64(e, 14) ^ ror64(e, 18) ^ ror64(e, 41);
            uint64_t ch = (e & f) ^ (~e & g);
            uint64_t t1 = hh + S1 + ch + SHA512_K[r + i] + w[i];
            uint64_t S0 = ror64(a, 28) ^ ror64(a, 34) ^ ror64(a, 39);
            uint64_t mj = (a & b) ^ (a & c) ^ (b & c);
            uint64_t t2 = S0 + mj;
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// ---------------------------------------------------------------- SHA-256 (FIPS 180-4)
static __device__ __constant__ uint32_t SHA256_K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

__device__ __forceinline__ uint32_t ror32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// One SHA-256 compression with the block in registers (16 big-endian words, static indices), as sha512_compress_regs.
__device__ __forceinline__ void sha256_compress_regs(uint32_t h[8], uint32_t w[16])
{
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
    for (int r = 0; r < 64; r += 16) {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (r) {
                uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
                uint32_t s0 = ror32(w15, 7) ^ ror32(w15, 18) ^ (w15 >> 3);
                uint32_t s1 = ror32(w2, 17) ^ ror32(w2, 19) ^ (w2 >> 10);
                w[i] = w[i] + s0 + w[(i + 9) & 15] + s1;
            }
            uint32_t S1 = ror32(e, 6) ^ ror32(e, 11) ^ ror32(e, 25);
            uint32_t ch = (e & f) ^ (~e & g);
            uint32_t t1 = hh + S1 + ch + SHA256_K[r + i] + w[i];
            uint32_t S0 = ror32(a, 2) ^ ror32(a, 13) ^ ror32(a, 22);
            uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
            uint32_t t2 = S0 + mj;
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// A public prefix hashed before the register strings: Ed25519ph's dom2(1, C) = "SigEd25519 no Ed25519 collisions" || 1 ||
// |C| || C (RFC 8032 5.1; ed25519-dalek signing.rs:945-951, verifying.rs:530-535), at most 34 + 255 bytes.  Travels as a
// __grid_constant__ kernel parameter, like the DST of hash_to_curve.cu.
#define SHA512_PREFIX_MAX 289
struct Sha512Prefix {
    uint8_t b[SHA512_PREFIX_MAX + 7];
    uint32_t len;
};

// dom2(1, context) for a context of at most 255 bytes (the caller checks the length)
static inline void ed25519ph_dom2(Sha512Prefix &d, const uint8_t *context, size_t context_len)
{
    const char *tag = "SigEd25519 no Ed25519 collisions";
    d = Sha512Prefix{};
    for (int j = 0; j < 32; j++) d.b[j] = (uint8_t)tag[j];
    d.b[32] = 1;                                                  // phflag
    d.b[33] = (uint8_t)context_len;
    for (size_t j = 0; j < context_len; j++) d.b[34 + j] = context[j];
    d.len = (uint32_t)(34 + context_len);
}

// SHA-512(P || X || M) with the blocks assembled in registers: P the public prefix (PRE = 1: `plen` bytes at `pre`;
// PRE = 0: none), X = NX register strings of 32 bytes (X0, then X1 when NX = 2; eight little-endian words each, their
// bytes in order), M = `len` bytes at `msg` (any alignment).  dig: 16 LE words.  Where each byte comes from depends on
// the lengths only, so X may be secret (the signer's nonce prefix).  With PRE = 0, X starts the first block at a fixed
// word index; with a prefix, X is shifted by plen mod 8 bytes once and each word of the first blocks takes its X part
// by a masked select over the shifted words (no register array is indexed at run time).
template <int NX, int PRE>
__device__ __forceinline__ void sha512_pxm(uint32_t dig[16], const uint8_t *pre, uint32_t plen, const uint32_t X0[8],
                                           const uint32_t X1[8], const uint8_t *__restrict__ msg, size_t len)
{
    uint64_t h[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                     0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
    // big-endian 64-bit word from two LE 32-bit words holding 8 consecutive bytes
#define SHA_BE64(lo, hi) (((uint64_t)__byte_perm((lo), 0, 0x0123) << 32) | (uint64_t)__byte_perm((hi), 0, 0x0123))
    if (!PRE) {
        const size_t total = 32 * NX + len;                      // message bytes of the hash input
        const size_t nblocks = (total + 1 + 16 + 127) / 128;
#pragma unroll 1
        for (size_t blk = 0; blk < nblocks; blk++) {
            uint64_t w[16];
            const size_t base = blk * 128;
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const size_t off = base + 8 * j;                 // first input byte of this word
                uint64_t v;
                if (blk == 0 && j < 4) v = SHA_BE64(X0[2 * j], X0[2 * j + 1]);
                else if (NX == 2 && blk == 0 && j < 8) v = SHA_BE64(X1[2 * (j - 4)], X1[2 * (j - 4) + 1]);
                else {
                    v = 0;
                    if (off + 8 <= total) {                      // eight message bytes
#pragma unroll
                        for (int b = 0; b < 8; b++) v = (v << 8) | (uint64_t)msg[off - 32 * NX + b];
                    } else if (off <= total) {                   // tail of the message, then the 0x80 marker
#pragma unroll
                        for (int b = 0; b < 8; b++) {
                            const size_t q = off + b;
                            const uint64_t byte = q < total ? (uint64_t)msg[q - 32 * NX] : (q == total ? 0x80u : 0u);
                            v = (v << 8) | byte;
                        }
                    }
                }
                w[j] = v;
            }
            if (blk == nblocks - 1) w[15] = (uint64_t)total * 8; // bit length (w[14] stays 0: inputs < 2^61 bytes)
            sha512_compress_regs(h, w);
        }
    } else {
        const size_t mstart = plen + 32 * NX, total = mstart + len;
        const size_t nblocks = (total + 1 + 16 + 127) / 128;
        const uint32_t sh = 8 * (plen & 7), w0 = plen >> 3;      // X starts sh bits into word w0 of the input
        uint64_t XS[4 * NX + 1];                                 // X shifted right by sh bits, as input words w0..w0+4NX
        {
            uint64_t XW[4 * NX];
#pragma unroll
            for (int k = 0; k < 4; k++) XW[k] = SHA_BE64(X0[2 * k], X0[2 * k + 1]);
#pragma unroll
            for (int k = 4; k < 4 * NX; k++) XW[k] = SHA_BE64(X1[2 * (k - 4)], X1[2 * (k - 4) + 1]);
#pragma unroll
            for (int k = 0; k <= 4 * NX; k++) {
                const uint64_t hi = k < 4 * NX ? XW[k] >> sh : 0;
                const uint64_t lo = k ? (XW[k - 1] << (56 - sh)) << 8 : 0;   // << (64 - sh), 0 when sh = 0
                XS[k] = hi | lo;
            }
        }
#pragma unroll 1
        for (size_t blk = 0; blk < nblocks; blk++) {
            uint64_t w[16];
            const size_t base = blk * 128;
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const size_t off = base + 8 * j, g = off >> 3;
                uint64_t v = 0;
                if (off + 8 <= plen) {                           // eight prefix bytes
#pragma unroll
                    for (int b = 0; b < 8; b++) v = (v << 8) | (uint64_t)pre[off + b];
                } else if (off >= mstart && off + 8 <= total) {  // eight message bytes
#pragma unroll
                    for (int b = 0; b < 8; b++) v = (v << 8) | (uint64_t)msg[off - mstart + b];
                } else if (off < total + 1) {                    // prefix / X / message / 0x80 boundaries
                    uint64_t xm = 0;                             // byte mask of X in this word
#pragma unroll
                    for (int b = 0; b < 8; b++) {
                        const size_t q = off + b;
                        const uint64_t byte = q < plen ? (uint64_t)pre[q]
                                              : q < mstart ? 0u
                                              : q < total ? (uint64_t)msg[q - mstart] : (q == total ? 0x80u : 0u);
                        v = (v << 8) | byte;
                        xm = (xm << 8) | (q >= plen && q < mstart ? 0xffu : 0u);
                    }
                    uint64_t xv = 0;
#pragma unroll
                    for (int k = 0; k <= 4 * NX; k++) xv |= XS[k] & (0ULL - (uint64_t)(g == w0 + (size_t)k));
                    v |= xv & xm;
                }
                w[j] = v;
            }
            if (blk == nblocks - 1) w[15] = (uint64_t)total * 8;
            sha512_compress_regs(h, w);
        }
    }
#undef SHA_BE64
#pragma unroll
    for (int i = 0; i < 8; i++) {
        dig[2 * i] = __byte_perm((uint32_t)(h[i] >> 32), 0, 0x0123);
        dig[2 * i + 1] = __byte_perm((uint32_t)h[i], 0, 0x0123);
    }
}

// SHA-512(R || A || M): the hash of batch.rs:179-191 / verifying.rs:515-523, one call per signature.
__device__ __forceinline__ void sha512_ram(uint32_t dig[16], const uint32_t R[8], const uint32_t A[8], const uint8_t *__restrict__ msg,
                                           size_t len)
{
    sha512_pxm<2, 0>(dig, nullptr, 0, R, A, msg, len);
}

// ---------------------------------------------------------------- Keccak-f[1600]
static __device__ __constant__ uint64_t KECCAK_RC[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
    0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
    0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
    0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
    0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};

__device__ __forceinline__ uint64_t rol64(uint64_t x, int n) { return (x << n) | (x >> (64 - n)); }

static __device__ __noinline__ void keccak_f1600(uint64_t *st)
{
    uint64_t a[25];
#pragma unroll
    for (int i = 0; i < 25; i++) a[i] = st[i];
#pragma unroll 1
    for (int round = 0; round < 24; round++) {
        uint64_t C0 = a[0] ^ a[5] ^ a[10] ^ a[15] ^ a[20];
        uint64_t C1 = a[1] ^ a[6] ^ a[11] ^ a[16] ^ a[21];
        uint64_t C2 = a[2] ^ a[7] ^ a[12] ^ a[17] ^ a[22];
        uint64_t C3 = a[3] ^ a[8] ^ a[13] ^ a[18] ^ a[23];
        uint64_t C4 = a[4] ^ a[9] ^ a[14] ^ a[19] ^ a[24];
        uint64_t D0 = C4 ^ rol64(C1, 1), D1 = C0 ^ rol64(C2, 1), D2 = C1 ^ rol64(C3, 1);
        uint64_t D3 = C2 ^ rol64(C4, 1), D4 = C3 ^ rol64(C0, 1);
#pragma unroll
        for (int y = 0; y < 25; y += 5) { a[y] ^= D0; a[y + 1] ^= D1; a[y + 2] ^= D2; a[y + 3] ^= D3; a[y + 4] ^= D4; }
        // rho + pi: B[y + 5*((2x+3y)%5)] = rol(a[x+5y], ROT[x+5y])
        uint64_t B[25];
        B[0] = a[0];
        B[10] = rol64(a[1], 1);   B[20] = rol64(a[2], 62);  B[5] = rol64(a[3], 28);   B[15] = rol64(a[4], 27);
        B[16] = rol64(a[5], 36);  B[1] = rol64(a[6], 44);   B[11] = rol64(a[7], 6);   B[21] = rol64(a[8], 55);  B[6] = rol64(a[9], 20);
        B[7] = rol64(a[10], 3);   B[17] = rol64(a[11], 10); B[2] = rol64(a[12], 43);  B[12] = rol64(a[13], 25); B[22] = rol64(a[14], 39);
        B[23] = rol64(a[15], 41); B[8] = rol64(a[16], 45);  B[18] = rol64(a[17], 15); B[3] = rol64(a[18], 21);  B[13] = rol64(a[19], 8);
        B[14] = rol64(a[20], 18); B[24] = rol64(a[21], 2);  B[9] = rol64(a[22], 61);  B[19] = rol64(a[23], 56); B[4] = rol64(a[24], 14);
#pragma unroll
        for (int y = 0; y < 25; y += 5) {
            a[y] = B[y] ^ (~B[y + 1] & B[y + 2]);
            a[y + 1] = B[y + 1] ^ (~B[y + 2] & B[y + 3]);
            a[y + 2] = B[y + 2] ^ (~B[y + 3] & B[y + 4]);
            a[y + 3] = B[y + 3] ^ (~B[y + 4] & B[y]);
            a[y + 4] = B[y + 4] ^ (~B[y] & B[y + 1]);
        }
        a[0] ^= KECCAK_RC[round];
    }
#pragma unroll
    for (int i = 0; i < 25; i++) st[i] = a[i];
}

// ---------------------------------------------------------------- STROBE-128 subset
#define STROBE_R 166u
#define SFLAG_I 1u
#define SFLAG_A 2u
#define SFLAG_C 4u
#define SFLAG_M 16u
#define SFLAG_K 32u

struct strobe128 {
    uint64_t st[25];
    uint32_t pos, pos_begin;
};

__device__ __forceinline__ void strobe_xor_byte(strobe128 &s, uint32_t idx, uint32_t v) { s.st[idx >> 3] ^= (uint64_t)v << (8 * (idx & 7)); }
__device__ __forceinline__ uint32_t strobe_get_byte(const strobe128 &s, uint32_t idx) { return (uint32_t)(s.st[idx >> 3] >> (8 * (idx & 7))) & 0xff; }
__device__ __forceinline__ void strobe_set_byte(strobe128 &s, uint32_t idx, uint32_t v)
{
    uint32_t sh = 8 * (idx & 7);
    s.st[idx >> 3] = (s.st[idx >> 3] & ~(0xffULL << sh)) | ((uint64_t)v << sh);
}

__device__ __forceinline__ void strobe_run_f(strobe128 &s)
{
    strobe_xor_byte(s, s.pos, s.pos_begin);
    strobe_xor_byte(s, s.pos + 1, 0x04);
    strobe_xor_byte(s, STROBE_R + 1, 0x80);
    keccak_f1600(s.st);
    s.pos = 0; s.pos_begin = 0;
}
__device__ __forceinline__ void strobe_absorb_byte(strobe128 &s, uint32_t v)
{
    strobe_xor_byte(s, s.pos, v);
    if (++s.pos == STROBE_R) strobe_run_f(s);
}
__device__ __forceinline__ void strobe_begin_op(strobe128 &s, uint32_t flags)
{
    uint32_t old_begin = s.pos_begin;
    s.pos_begin = s.pos + 1;
    strobe_absorb_byte(s, old_begin);
    strobe_absorb_byte(s, flags);
    if ((flags & (SFLAG_C | SFLAG_K)) && s.pos != 0) strobe_run_f(s);
}
__device__ __forceinline__ void strobe_init(strobe128 &s, const uint8_t *proto, uint32_t len)
{
#pragma unroll
    for (int i = 0; i < 25; i++) s.st[i] = 0;
    const uint8_t init[18] = {1, STROBE_R + 2, 1, 0, 1, 96, 'S', 'T', 'R', 'O', 'B', 'E', 'v', '1', '.', '0', '.', '2'};
    for (uint32_t i = 0; i < 18; i++) strobe_xor_byte(s, i, init[i]);
    keccak_f1600(s.st);
    s.pos = 0; s.pos_begin = 0;
    strobe_begin_op(s, SFLAG_M | SFLAG_A);
    for (uint32_t i = 0; i < len; i++) strobe_absorb_byte(s, proto[i]);
}
// Merlin append_message (transcript.rs:69-74) with the message given as LE 32-bit words
__device__ __forceinline__ void merlin_append_words(strobe128 &s, const uint8_t *label, uint32_t llen,
                                                    const uint32_t *words, uint32_t nbytes)
{
    strobe_begin_op(s, SFLAG_M | SFLAG_A);
    for (uint32_t i = 0; i < llen; i++) strobe_absorb_byte(s, label[i]);
    strobe_absorb_byte(s, nbytes & 0xff); strobe_absorb_byte(s, (nbytes >> 8) & 0xff);   // meta_ad(len, more=true)
    strobe_absorb_byte(s, (nbytes >> 16) & 0xff); strobe_absorb_byte(s, nbytes >> 24);
    strobe_begin_op(s, SFLAG_A);
    for (uint32_t i = 0; i < nbytes; i++) strobe_absorb_byte(s, (words[i >> 2] >> (8 * (i & 3))) & 0xff);
}
