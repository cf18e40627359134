// Host build of the device hash-to-group code (elligator.cuh over fe.cuh / fe64.cuh / ge.cuh) with the limb-bound
// assertions of fe.cuh and the operand-scale assertions of fe64.cuh enabled, exported with a tiny C ABI for
// tests/test_hash_to_curve_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product.  The library's kernels compress SHA-512 blocks with
// hash.cuh's sha512_compress_regs; this build supplies a FIPS 180-4 compression function of its own for the same role.
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/elligator.cuh"
#include <string.h>

static const uint64_t K512[80] = {
    0x428a2f98d728ae22ULL, 0x7137449123ef65cdULL, 0xb5c0fbcfec4d3b2fULL, 0xe9b5dba58189dbbcULL, 0x3956c25bf348b538ULL,
    0x59f111f1b605d019ULL, 0x923f82a4af194f9bULL, 0xab1c5ed5da6d8118ULL, 0xd807aa98a3030242ULL, 0x12835b0145706fbeULL,
    0x243185be4ee4b28cULL, 0x550c7dc3d5ffb4e2ULL, 0x72be5d74f27b896fULL, 0x80deb1fe3b1696b1ULL, 0x9bdc06a725c71235ULL,
    0xc19bf174cf692694ULL, 0xe49b69c19ef14ad2ULL, 0xefbe4786384f25e3ULL, 0x0fc19dc68b8cd5b5ULL, 0x240ca1cc77ac9c65ULL,
    0x2de92c6f592b0275ULL, 0x4a7484aa6ea6e483ULL, 0x5cb0a9dcbd41fbd4ULL, 0x76f988da831153b5ULL, 0x983e5152ee66dfabULL,
    0xa831c66d2db43210ULL, 0xb00327c898fb213fULL, 0xbf597fc7beef0ee4ULL, 0xc6e00bf33da88fc2ULL, 0xd5a79147930aa725ULL,
    0x06ca6351e003826fULL, 0x142929670a0e6e70ULL, 0x27b70a8546d22ffcULL, 0x2e1b21385c26c926ULL, 0x4d2c6dfc5ac42aedULL,
    0x53380d139d95b3dfULL, 0x650a73548baf63deULL, 0x766a0abb3c77b2a8ULL, 0x81c2c92e47edaee6ULL, 0x92722c851482353bULL,
    0xa2bfe8a14cf10364ULL, 0xa81a664bbc423001ULL, 0xc24b8b70d0f89791ULL, 0xc76c51a30654be30ULL, 0xd192e819d6ef5218ULL,
    0xd69906245565a910ULL, 0xf40e35855771202aULL, 0x106aa07032bbd1b8ULL, 0x19a4c116b8d2d0c8ULL, 0x1e376c085141ab53ULL,
    0x2748774cdf8eeb99ULL, 0x34b0bcb5e19b48a8ULL, 0x391c0cb3c5c95a63ULL, 0x4ed8aa4ae3418acbULL, 0x5b9cca4f7763e373ULL,
    0x682e6ff3d6b2b8a3ULL, 0x748f82ee5defb2fcULL, 0x78a5636f43172f60ULL, 0x84c87814a1f0ab72ULL, 0x8cc702081a6439ecULL,
    0x90befffa23631e28ULL, 0xa4506cebde82bde9ULL, 0xbef9a3f7b2c67915ULL, 0xc67178f2e372532bULL, 0xca273eceea26619cULL,
    0xd186b8c721c0c207ULL, 0xeada7dd6cde0eb1eULL, 0xf57d4f7fee6ed178ULL, 0x06f067aa72176fbaULL, 0x0a637dc5a2c898a6ULL,
    0x113f9804bef90daeULL, 0x1b710b35131c471bULL, 0x28db77f523047d84ULL, 0x32caab7b40c72493ULL, 0x3c9ebe0a15c9bebcULL,
    0x431d67c49c100d4cULL, 0x4cc5d4becb3e42b6ULL, 0x597f299cfc657e2aULL, 0x5fcb6fab3ad6faecULL, 0x6c44198c4a475817ULL};

static inline uint64_t ror(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

void h2c_host_sha512_compress(uint64_t h[8], uint64_t w16[16])
{
    uint64_t w[80];
    for (int t = 0; t < 16; t++) w[t] = w16[t];
    for (int t = 16; t < 80; t++)
        w[t] = w[t - 16] + (ror(w[t - 15], 1) ^ ror(w[t - 15], 8) ^ (w[t - 15] >> 7)) + w[t - 7] +
               (ror(w[t - 2], 19) ^ ror(w[t - 2], 61) ^ (w[t - 2] >> 6));
    uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 80; t++) {
        uint64_t t1 = hh + (ror(e, 14) ^ ror(e, 18) ^ ror(e, 41)) + ((e & f) ^ (~e & g)) + K512[t] + w[t];
        uint64_t t2 = (ror(a, 28) ^ ror(a, 34) ^ ror(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

static void fe_out(uint8_t *out, const fe &f)
{
    uint32_t w[8];
    fe_tobytes_words(w, f);
    memcpy(out, w, 32);
}

static void fe_in(fe &f, const uint8_t *in)
{
    uint32_t w[8];
    memcpy(w, in, 32);
    fe_frombytes_words(f, w);
}

extern "C" {
// compress(elligator_ristretto_flavor(from_bytes(r0)))
void h_ristretto_elligator(uint8_t *out, const uint8_t *r0)
{
    fe r; fe_in(r, r0);
    ge_p3 P; ristretto_elligator(P, r);
    uint32_t w[8]; ristretto_compress<1>(w, P); memcpy(out, w, 32);
}

void h_from_uniform_bytes(uint8_t *out, const uint8_t *in)
{
    uint32_t w[16]; memcpy(w, in, 64);
    ge_p3 P; ristretto_from_uniform(P, w);
    uint32_t o[8]; ristretto_compress<1>(o, P); memcpy(out, o, 32);
}

void h_hash_from_bytes(uint8_t *out, const uint8_t *msg, size_t len)
{
    uint32_t o[8]; ristretto_hash_from_bytes(o, msg, len); memcpy(out, o, 32);
}

// uniform_bytes of expand_msg_xmd: 48 count bytes
void h_xmd(uint8_t *out, const uint8_t *msg, size_t len, const uint8_t *dst, uint32_t dlen, int count)
{
    uint64_t b1[8], b2[8];
    if (count == 2) xmd_sha512<2>(b1, b2, msg, len, dst, dlen); else xmd_sha512<1>(b1, b2, msg, len, dst, dlen);
    uint8_t buf[128];
    for (int i = 0; i < 64; i++) { buf[i] = (uint8_t)(b1[i >> 3] >> (56 - 8 * (i & 7))); buf[64 + i] = (uint8_t)(b2[i >> 3] >> (56 - 8 * (i & 7))); }
    memcpy(out, buf, 48 * count);
}

// hash_to_field::<Sha512, count>: count canonical 32-byte elements
void h_hash_to_field(uint8_t *out, const uint8_t *msg, size_t len, const uint8_t *dst, uint32_t dlen, int count)
{
    fe u[2];
    if (count == 2) h2c_hash_to_field<2>(u, msg, len, dst, dlen); else h2c_hash_to_field<1>(u, msg, len, dst, dlen);
    for (int i = 0; i < count; i++) fe_out(out + 32 * i, u[i]);
}

void h_from_bytes_wide(uint8_t *out, const uint8_t *in)
{
    uint32_t w[16]; memcpy(w, in, 64);
    fe r; h2c_from_bytes_wide(r, w); fe_out(out, r);
}

// elligator_encode(u): xn | xd | y, canonical
void h_ell2_encode(uint8_t *out, const uint8_t *u_bytes)
{
    fe u, xn, xd, y; fe_in(u, u_bytes);
    ell2_encode(xn, xd, y, u);
    fe_out(out, xn); fe_out(out + 32, xd); fe_out(out + 64, y);
}

// compress(map_to_curve(u)) (no cofactor clearing); returns the tv1 == 0 flag
int h_map_to_curve(uint8_t *out, const uint8_t *u_bytes)
{
    fe u; fe_in(u, u_bytes);
    ge_p3 P; ell2_map_to_curve(P, u);
    uint32_t o[8]; ge_compress<1>(o, P); memcpy(out, o, 32);
    fe xMn, xMd, yMn, xd, yd, tv1;
    ell2_encode(xMn, xMd, yMn, u);
    fe_mul(xd, xMd, yMn); fe_add(yd, xMn, xMd); fe_mul(tv1, xd, yd);
    return fe_iszero(tv1);
}

void h_hash_to_curve(uint8_t *out, const uint8_t *msg, size_t len, const uint8_t *dst, uint32_t dlen, int count)
{
    uint32_t o[8];
    if (count == 2) edwards_hash_to_curve<2>(o, msg, len, dst, dlen); else edwards_hash_to_curve<1>(o, msg, len, dst, dlen);
    memcpy(out, o, 32);
}
}
