// Host build of the device Lizard code (lizard.cuh over elligator.cuh / fe.cuh / fe64.cuh / ge.cuh) with the limb-bound
// assertions of fe.cuh and the operand-scale assertions of fe64.cuh enabled, exported with a tiny C ABI for
// tests/test_lizard_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product.  The kernels compress SHA-256 blocks with hash.cuh's
// sha256_compress_regs; this build supplies a FIPS 180-4 compression of its own for the same role, and a table of fake
// digests: a one-block hash of 16 data bytes listed in the table gets the listed digest instead.  That reaches decode
// states no real input reaches (two candidates of one point that both pass the tag check, about 2^-122).
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/lizard.cuh"
#include <string.h>

#include <vector>

static const uint32_t K256[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u,
    0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u,
    0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u,
    0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u,
    0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, 0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u,
    0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au,
    0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u,
    0xc67178f2u};

static inline uint32_t ror(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

struct FakeDigest { uint32_t block[16]; uint32_t h[8]; };
static std::vector<FakeDigest> g_fakes;

static bool is_iv(const uint32_t h[8])
{
    static const uint32_t iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    return memcmp(h, iv, 32) == 0;
}

void lizard_host_sha256_compress(uint32_t h[8], uint32_t w16[16])
{
    if (is_iv(h))
        for (const FakeDigest &f : g_fakes)
            if (memcmp(f.block, w16, 64) == 0) { memcpy(h, f.h, 32); return; }
    uint32_t w[64];
    for (int t = 0; t < 16; t++) w[t] = w16[t];
    for (int t = 16; t < 64; t++)
        w[t] = w[t - 16] + (ror(w[t - 15], 7) ^ ror(w[t - 15], 18) ^ (w[t - 15] >> 3)) + w[t - 7] +
               (ror(w[t - 2], 17) ^ ror(w[t - 2], 19) ^ (w[t - 2] >> 10));
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 64; t++) {
        uint32_t t1 = hh + (ror(e, 6) ^ ror(e, 11) ^ ror(e, 25)) + ((e & f) ^ (~e & g)) + K256[t] + w[t];
        uint32_t t2 = (ror(a, 2) ^ ror(a, 13) ^ ror(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// the kernels' point loading (csrc/point_load.cuh) for fmt 2 (CompressedRistretto) and 1 (20 radix-2^51 limbs)
static uint32_t load_point(ge_p3 &P, const uint8_t *pt, int fmt)
{
    if (fmt == 1) {
        uint64_t l[20];
        memcpy(l, pt, 160);
        fe_from_limbs51(P.X, l); fe_from_limbs51(P.Y, l + 5); fe_from_limbs51(P.Z, l + 10); fe_from_limbs51(P.T, l + 15);
        return 1;
    }
    uint32_t s[8];
    memcpy(s, pt, 32);
    const uint32_t good = ristretto_decompress<1>(P, s);
    ge_p3 id; ge_p3_identity(id);
    fe_cmov(P.X, id.X, 1u - good); fe_cmov(P.Y, id.Y, 1u - good); fe_cmov(P.Z, id.Z, 1u - good); fe_cmov(P.T, id.T, 1u - good);
    return good;
}

extern "C" {
// one-block SHA-256 of 16 bytes, as the kernels compute it (digest bytes)
void h_sha256_16(uint8_t *out, const uint8_t *data)
{
    uint32_t d[4], dig[8];
    memcpy(d, data, 16);
    lizard_sha256_16(dig, d);
    memcpy(out, dig, 32);
}

void h_map_to_curve(uint8_t *out, const uint8_t *in)
{
    uint32_t w[8], o[8];
    memcpy(w, in, 32);
    ristretto_map_to_curve(o, w);
    memcpy(out, o, 32);
}

void h_lizard_encode(uint8_t *out, const uint8_t *data)
{
    uint32_t d[4], o[8];
    memcpy(d, data, 16);
    lizard_encode(o, d);
    memcpy(out, o, 32);
}

// returns n_found, or -1 for an undecodable encoding (the kernel's status 2); data zero unless n_found == 1
int h_lizard_decode(uint8_t *data, const uint8_t *pt, int fmt)
{
    ge_p3 P;
    const uint32_t good = load_point(P, pt, fmt);
    uint32_t d[4];
    const uint32_t n_found = lizard_decode(d, P);
    memcpy(data, d, 16);
    return good ? (int)n_found : -1;
}

// returns the mask, or -1 for an undecodable encoding; out 16 x 32 bytes
int h_map_to_curve_inverse(uint8_t *out, const uint8_t *pt, int fmt)
{
    ge_p3 P;
    const uint32_t good = load_point(P, pt, fmt);
    const uint32_t m = map_to_curve_inverse(P, [&](uint32_t j, const uint32_t b[8], uint32_t) { memcpy(out + 32 * j, b, 32); });
    return good ? (int)m : -1;
}

// the four Jacobi points (S0, T0, ..., S3, T3), canonical
void h_to_jacobi(uint8_t *out, const uint8_t *pt, int fmt)
{
    ge_p3 P;
    (void)load_point(P, pt, fmt);
    fe S[4], T[4];
    ristretto_to_jacobi(S, T, P);
    for (int k = 0; k < 4; k++) {
        uint32_t w[8];
        fe_tobytes_words(w, S[k]); memcpy(out + 64 * k, w, 32);
        fe_tobytes_words(w, T[k]); memcpy(out + 64 * k + 32, w, 32);
    }
}

// e_inv_positive(s, t): returns is_some, out the value (zero when None)
int h_e_inv_positive(uint8_t *out, const uint8_t *s_bytes, const uint8_t *t_bytes)
{
    uint32_t w[8];
    fe s, t, x;
    memcpy(w, s_bytes, 32); fe_frombytes_words(s, w);
    memcpy(w, t_bytes, 32); fe_frombytes_words(t, w);
    const uint32_t def = jacobi_e_inv_positive(x, s, t);
    fe_tobytes_words(w, x);
    memcpy(out, w, 32);
    return (int)def;
}

// from now on, the one-block hash of these 16 bytes is this 32-byte digest
void h_fake_digest(const uint8_t *data, const uint8_t *digest)
{
    FakeDigest f;
    uint32_t d[4];
    memcpy(d, data, 16);
    for (int k = 0; k < 4; k++) f.block[k] = h2c_bswap32(d[k]);
    f.block[4] = 0x80000000u;
    for (int k = 5; k < 15; k++) f.block[k] = 0;
    f.block[15] = 128;
    for (int k = 0; k < 8; k++)
        f.h[k] = (uint32_t)digest[4 * k] << 24 | (uint32_t)digest[4 * k + 1] << 16 | (uint32_t)digest[4 * k + 2] << 8 | digest[4 * k + 3];
    g_fakes.push_back(f);
}

void h_fake_clear() { g_fakes.clear(); }
}
