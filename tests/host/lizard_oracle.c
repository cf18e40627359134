/*
 * lizard_oracle.c -- CPU restatement of the reference's Lizard encoding and decoding and of the inverse of the Ristretto
 * Elligator map, on the oracle's radix-2^51 field.  TEST INFRASTRUCTURE: the parity source of the GPU Lizard paths and the
 * CPU baseline of tools/bench_lizard.py.  Built together with tests/host/h2c_oracle.c (whose h2c_ristretto_elligator is the
 * forward map) and the oracle library's sources (tests/lizard_oracle.py); neither is changed.
 *
 *   C/ristretto/elligator.rs:62-67       RistrettoPoint::map_to_curve (h2c_ristretto_elligator)
 *   C/lizard/lizard_ristretto.rs:25-71   lizard_encode / lizard_decode::<Sha256>
 *   C/lizard/lizard_ristretto.rs:78-219  elligator_ristretto_flavor_inverse, to_jacobi_quartic_ristretto, map_to_curve_inverse
 *   C/lizard/jacobi_quartic.rs:28-70     JacobiPoint::e_inv_positive, dual
 * The digest is SHA-256 (FIPS 180-4, below).  Decode hashes all 16 candidates, as the reference does.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

void h2c_ristretto_elligator(uint8_t out[32], const uint8_t r0[32]);   /* tests/host/h2c_oracle.c */

/* constants as canonical little-endian encodings (lizard_constants.rs:25-46); tests/test_lizard_golden.py checks each
 * Lizard constant against its definition */
enum { LZ_SQRT_ID, LZ_DP1_OVER_DM1, LZ_MDOUBLE_INVSQRT_A_MINUS_D, LZ_MIDOUBLE_INVSQRT_A_MINUS_D, LZ_MINVSQRT_ONE_PLUS_D, LZ_SQRT_M1,
       LZ_MINUS_ONE, LZ_COUNT };
static const uint8_t LZB[LZ_COUNT][32] = {
    /* SQRT_ID */
    {0xa8, 0x1b, 0x5c, 0x4a, 0xcb, 0x2a, 0x30, 0x75, 0xaa, 0x6d, 0xea, 0x0e, 0x2d, 0xa9, 0xbc, 0xcd,
     0x15, 0x6e, 0xeb, 0x73, 0x99, 0x54, 0x34, 0x75, 0x97, 0xeb, 0x7b, 0xf4, 0x58, 0x55, 0xb3, 0x05},
    /* DP1_OVER_DM1 */
    {0x2c, 0xbb, 0x81, 0x9b, 0x5f, 0xac, 0x7f, 0x27, 0xc8, 0x1d, 0x24, 0xcd, 0xf1, 0xe7, 0x9a, 0x48,
     0x24, 0x18, 0x9f, 0x99, 0x5f, 0xd9, 0xf8, 0xae, 0x9d, 0xd8, 0xe8, 0xa7, 0x30, 0xc8, 0x67, 0x0e},
    /* MDOUBLE_INVSQRT_A_MINUS_D */
    {0x06, 0x7e, 0x45, 0xff, 0xaa, 0x04, 0x6e, 0xcc, 0x82, 0x1a, 0x7d, 0x4b, 0xd1, 0xd3, 0xa1, 0xc5,
     0x7e, 0x4f, 0xfc, 0x03, 0xdc, 0x08, 0x7b, 0xd2, 0xbb, 0x06, 0xa0, 0x60, 0xf4, 0xed, 0x26, 0x0f},
    /* MIDOUBLE_INVSQRT_A_MINUS_D */
    {0xd8, 0xbb, 0x77, 0x63, 0x10, 0xb7, 0x5d, 0x16, 0x9c, 0x6c, 0xb5, 0xd7, 0x38, 0xee, 0xa5, 0x9c,
     0x10, 0x59, 0x0b, 0x28, 0x85, 0x58, 0xe0, 0x3d, 0x50, 0x3d, 0x56, 0x06, 0x68, 0x0b, 0x1b, 0x14},
    /* MINVSQRT_ONE_PLUS_D */
    {0x01, 0x22, 0x44, 0xce, 0x77, 0x24, 0xd1, 0xf4, 0xb1, 0x49, 0x25, 0x94, 0xe3, 0x08, 0xad, 0xb1,
     0x77, 0x53, 0xfa, 0x6b, 0xbd, 0xd3, 0x0f, 0xe1, 0x57, 0xe1, 0xd4, 0xfc, 0x4b, 0x7a, 0xf2, 0x75},
    /* SQRT_M1 */
    {0xb0, 0xa0, 0x0e, 0x4a, 0x27, 0x1b, 0xee, 0xc4, 0x78, 0xe4, 0x2f, 0xad, 0x06, 0x18, 0x43, 0x2f,
     0xa7, 0xd7, 0xfb, 0x3d, 0x99, 0x00, 0x4d, 0x2b, 0x0b, 0xdf, 0xc1, 0x4f, 0x80, 0x24, 0x83, 0x2b},
    /* MINUS_ONE */
    {0xec, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
     0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x7f},
};

static void LZK(fe51 *o, int k) { fe_from_bytes(o, LZB[k]); }

void lz_constant(uint8_t out[32], int k) { memcpy(out, LZB[k], 32); }

/* ---- SHA-256, FIPS 180-4 ---- */
static const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

static uint32_t ror32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

static void sha256_block(uint32_t h[8], const uint8_t blk[64])
{
    uint32_t w[64];
    for (int t = 0; t < 16; t++)
        w[t] = (uint32_t)blk[4 * t] << 24 | (uint32_t)blk[4 * t + 1] << 16 | (uint32_t)blk[4 * t + 2] << 8 | blk[4 * t + 3];
    for (int t = 16; t < 64; t++)
        w[t] = w[t - 16] + (ror32(w[t - 15], 7) ^ ror32(w[t - 15], 18) ^ (w[t - 15] >> 3)) + w[t - 7] +
               (ror32(w[t - 2], 17) ^ ror32(w[t - 2], 19) ^ (w[t - 2] >> 10));
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 64; t++) {
        uint32_t t1 = hh + (ror32(e, 6) ^ ror32(e, 11) ^ ror32(e, 25)) + ((e & f) ^ (~e & g)) + K256[t] + w[t];
        uint32_t t2 = (ror32(a, 2) ^ ror32(a, 13) ^ ror32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

void lz_sha256(uint8_t out[32], const uint8_t *msg, size_t len)
{
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    size_t off = 0;
    for (; off + 64 <= len; off += 64) sha256_block(h, msg + off);
    uint8_t blk[128] = {0};
    size_t rem = len - off;
    if (rem) memcpy(blk, msg + off, rem);
    blk[rem] = 0x80;
    size_t nb = rem + 1 + 8 <= 64 ? 1 : 2;
    uint64_t bits = (uint64_t)len * 8;
    for (int k = 0; k < 8; k++) blk[64 * nb - 1 - k] = (uint8_t)(bits >> (8 * k));
    for (size_t b = 0; b < nb; b++) sha256_block(h, blk + 64 * b);
    for (int k = 0; k < 8; k++) {
        out[4 * k] = (uint8_t)(h[k] >> 24); out[4 * k + 1] = (uint8_t)(h[k] >> 16);
        out[4 * k + 2] = (uint8_t)(h[k] >> 8); out[4 * k + 3] = (uint8_t)h[k];
    }
}

/* lizard_ristretto.rs:29-36: the digest with bytes 8..24 replaced by the data, bit 0 and the top two bits cleared */
static void lizard_tag(uint8_t out[32], const uint8_t data[16])
{
    lz_sha256(out, data, 16);
    memcpy(out + 8, data, 16);
    out[0] &= 0xfe;
    out[31] &= 0x3f;
}

/* RistrettoPoint::lizard_encode::<Sha256> -> CompressedRistretto */
void lz_encode(uint8_t out[32], const uint8_t data[16])
{
    uint8_t fe_bytes[32];
    lizard_tag(fe_bytes, data);
    h2c_ristretto_elligator(out, fe_bytes);                /* map_to_curve_restricted = map_to_curve (C/ristretto/elligator.rs:62-67) */
}

typedef struct { fe51 S, T; } jacobi_point;

/* to_jacobi_quartic_ristretto, lizard_ristretto.rs:117-188 */
static void to_jacobi_quartic_ristretto(jacobi_point jc[4], const ge_p3 *P)
{
    fe51 x2, y2, y4, z2, z_min_y, z_pl_y, z2_min_y2, t, gamma, den, s_over_x, sp_over_xp, tmp, c, iz, iz_min_x, iz_pl_x;
    fe51 s_over_y, sp_over_yp, sm1, one, m1;
    LZK(&sm1, LZ_SQRT_M1); fe_one(&one); LZK(&m1, LZ_MINUS_ONE);
    fe_square(&x2, &P->X); fe_square(&y2, &P->Y); fe_square(&y4, &y2); fe_square(&z2, &P->Z);
    fe_sub(&z_min_y, &P->Z, &P->Y); fe_add(&z_pl_y, &P->Z, &P->Y); fe_sub(&z2_min_y2, &z2, &y2);
    fe_mul(&t, &y4, &x2); fe_mul(&t, &t, &z2_min_y2);
    fe_invsqrt(&gamma, &t);
    fe_mul(&den, &gamma, &y2);
    fe_mul(&s_over_x, &den, &z_min_y); fe_mul(&sp_over_xp, &den, &z_pl_y);
    fe_mul(&jc[0].S, &s_over_x, &P->X);
    fe_neg(&t, &sp_over_xp); fe_mul(&jc[1].S, &t, &P->X);
    LZK(&c, LZ_MDOUBLE_INVSQRT_A_MINUS_D); fe_mul(&tmp, &c, &P->Z);
    fe_mul(&jc[0].T, &tmp, &s_over_x); fe_mul(&jc[1].T, &tmp, &sp_over_xp);
    fe_neg(&t, &z2_min_y2); LZK(&c, LZ_MINVSQRT_ONE_PLUS_D); fe_mul(&t, &t, &c); fe_mul(&den, &t, &gamma);
    fe_mul(&iz, &sm1, &P->Z); fe_sub(&iz_min_x, &iz, &P->X); fe_add(&iz_pl_x, &iz, &P->X);
    fe_mul(&s_over_y, &den, &iz_min_x); fe_mul(&sp_over_yp, &den, &iz_pl_x);
    fe_mul(&jc[2].S, &s_over_y, &P->Y);
    fe_neg(&t, &sp_over_yp); fe_mul(&jc[3].S, &t, &P->Y);
    LZK(&c, LZ_MDOUBLE_INVSQRT_A_MINUS_D); fe_mul(&tmp, &c, &iz);
    fe_mul(&jc[2].T, &tmp, &s_over_y); fe_mul(&jc[3].T, &tmp, &sp_over_yp);
    int xy0 = fe_is_zero(&P->X) | fe_is_zero(&P->Y);
    LZK(&c, LZ_MIDOUBLE_INVSQRT_A_MINUS_D);
    fe_cond_assign(&jc[0].T, &one, xy0); fe_cond_assign(&jc[1].T, &one, xy0);
    fe_cond_assign(&jc[2].T, &c, xy0); fe_cond_assign(&jc[3].T, &c, xy0);
    fe_cond_assign(&jc[2].S, &one, xy0); fe_cond_assign(&jc[3].S, &m1, xy0);
}

/* JacobiPoint::e_inv_positive, jacobi_quartic.rs:28-63; returns is_some */
static int e_inv_positive(fe51 *out, const jacobi_point *jp)
{
    fe51 one, c, a, a2, s2, s4, t, y, pms2, x;
    fe_one(&one); fe_zero(out);
    int s_is_zero = fe_is_zero(&jp->S), t_equals_one = fe_ct_eq(&jp->T, &one);
    LZK(&c, LZ_SQRT_ID); fe_cond_assign(out, &c, t_equals_one);
    int is_defined = s_is_zero, done = s_is_zero;
    fe_add(&t, &jp->T, &one); LZK(&c, LZ_DP1_OVER_DM1); fe_mul(&a, &t, &c);
    fe_square(&a2, &a);
    fe_square(&s2, &jp->S); fe_square(&s4, &s2);
    fe_sub(&t, &s4, &a2); LZK(&c, LZ_SQRT_M1); fe_mul(&t, &t, &c);
    int sq = fe_invsqrt(&y, &t);
    is_defined |= sq; done |= !sq;
    pms2 = s2; fe_cond_negate(&pms2, fe_is_negative(&jp->S));
    fe_add(&t, &a, &pms2); fe_mul(&x, &t, &y);
    fe_cond_negate(&x, fe_is_negative(&x));
    fe_cond_assign(out, &x, !done);
    return is_defined;
}

/* elligator_ristretto_flavor_inverse, lizard_ristretto.rs:78-110: fes[16], some[16] */
static void elligator_inverse(fe51 fes[16], int some[16], const ge_p3 *P)
{
    jacobi_point jc[4];
    to_jacobi_quartic_ristretto(jc, P);
    for (int k = 0; k < 4; k++) {
        jacobi_point dual;
        fe_neg(&dual.S, &jc[k].S); fe_neg(&dual.T, &jc[k].T);
        some[2 * k] = e_inv_positive(&fes[2 * k], &jc[k]);
        some[2 * k + 1] = e_inv_positive(&fes[2 * k + 1], &dual);
    }
    for (int j = 0; j < 8; j++) { fe_neg(&fes[8 + j], &fes[j]); some[8 + j] = some[j]; }
}

/* a point of the C ABI's formats: fmt 2 CompressedRistretto, 1 twenty radix-2^51 limbs (as given); 1 if it decodes */
static int lz_load(ge_p3 *P, const uint8_t *pt, int fmt)
{
    if (fmt == 1) {
        uint64_t l[20]; memcpy(l, pt, 160); ge_p3_from_limbs(P, l); return 1;
    }
    return ristretto_decompress(P, pt);
}

/* RistrettoPoint::lizard_decode::<Sha256>: 0 Some, 1 None, 2 undecodable; data zero unless 0.  n_found_out (optional) */
int lz_decode(uint8_t data[16], const uint8_t *pt, int fmt, int *n_found_out)
{
    ge_p3 P;
    memset(data, 0, 16);
    if (!lz_load(&P, pt, fmt)) { if (n_found_out) *n_found_out = 0; return 2; }
    fe51 fes[16]; int some[16];
    elligator_inverse(fes, some, &P);
    uint8_t result[16] = {0};
    int n_found = 0;
    for (int j = 0; j < 16; j++) {
        fe51 z; fe_zero(&z);
        fe51 fe = fes[j]; fe_cond_assign(&fe, &z, !some[j]);
        uint8_t bytes[32], expected[32];
        fe_to_bytes(bytes, &fe);
        lizard_tag(expected, bytes + 8);
        int ok = some[j] && memcmp(expected, bytes, 32) == 0;
        if (ok) memcpy(result, bytes + 8, 16);
        n_found += ok;
    }
    if (n_found_out) *n_found_out = n_found;
    if (n_found != 1) return 1;
    memcpy(data, result, 16);
    return 0;
}

/* RistrettoPoint::map_to_curve_inverse: out 16 x 32 (zeros where None), *mask; returns 1 if the encoding does not decode */
int lz_map_to_curve_inverse(uint8_t out[512], uint16_t *mask, const uint8_t *pt, int fmt)
{
    ge_p3 P;
    memset(out, 0, 512); *mask = 0;
    if (!lz_load(&P, pt, fmt)) return 1;
    fe51 fes[16]; int some[16];
    elligator_inverse(fes, some, &P);
    for (int j = 0; j < 16; j++)
        if (some[j]) { fe_to_bytes(out + 32 * j, &fes[j]); *mask |= (uint16_t)(1u << j); }
    return 0;
}

void lz_encode_batch(uint8_t *out, const uint8_t *data, size_t n)
{
    for (size_t i = 0; i < n; i++) lz_encode(out + 32 * i, data + 16 * i);
}

void lz_map_to_curve_batch(uint8_t *out, const uint8_t *in, size_t n)
{
    for (size_t i = 0; i < n; i++) h2c_ristretto_elligator(out + 32 * i, in + 32 * i);
}

void lz_decode_batch(uint8_t *data, uint8_t *status, const uint8_t *pts, int fmt, size_t n)
{
    const size_t w = fmt == 1 ? 160 : 32;
    for (size_t i = 0; i < n; i++) status[i] = (uint8_t)lz_decode(data + 16 * i, pts + w * i, fmt, NULL);
}

void lz_map_to_curve_inverse_batch(uint8_t *out, uint16_t *mask, const uint8_t *pts, int fmt, size_t n)
{
    const size_t w = fmt == 1 ? 160 : 32;
    for (size_t i = 0; i < n; i++) (void)lz_map_to_curve_inverse(out + 512 * i, mask + i, pts + w * i, fmt);
}
