/*
 * h2c_oracle.c -- CPU restatement of the reference's hashing into the group, on the oracle's radix-2^51 field.
 * TEST INFRASTRUCTURE: the parity source of the GPU hash-to-group paths and the CPU baseline of
 * tools/bench_hash_to_curve.py.  Built together with the oracle library's sources (tests/h2c_oracle.py), whose
 * fe_*, sha512_*, ge_*, ristretto_compress and ge_compress it uses; the oracle library itself is unchanged.
 *
 *   C/ristretto/elligator.rs:15-51   elligator_ristretto_flavor     C/ristretto.rs:736-790  hash_from_bytes, from_uniform_bytes
 *   C/field.rs:110-147               from_bytes_wide                C/field.rs:397-516      hash_to_field, expand_msg_xmd
 *   C/montgomery.rs:276-363          elligator_encode               C/edwards.rs:651-750    map_to_curve, encode/hash_to_curve
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

/* constants as canonical little-endian encodings; tests/test_hash_to_curve_golden.py checks each against its definition */
enum { K_ONE_MINUS_D_SQ, K_D_MINUS_ONE_SQ, K_SQRT_AD_MINUS_ONE, K_MINUS_ONE, K_MONT_A, K_MONT_A_NEG, K_SQRTAM2, K_ELL2_C2,
       K_D, K_SQRTM1, K_COUNT };
static const uint8_t KB[K_COUNT][32] = {
    /* ONE_MINUS_EDWARDS_D_SQUARED = 1 - d^2 */
    {0x76, 0xc1, 0x5f, 0x94, 0xc1, 0x09, 0x7c, 0xe2, 0x0f, 0x35, 0x5e, 0xcd, 0x38, 0xa1, 0x81, 0x2c,
     0xe4, 0xdf, 0x70, 0xbe, 0xdd, 0xab, 0x94, 0x99, 0xd7, 0xe0, 0xb3, 0xb2, 0xa8, 0x72, 0x90, 0x02},
    /* EDWARDS_D_MINUS_ONE_SQUARED = (d - 1)^2 */
    {0x20, 0x4d, 0xed, 0x44, 0xaa, 0x5a, 0xad, 0x31, 0x99, 0x19, 0x1e, 0xb0, 0x2c, 0x4a, 0x9e, 0xd2,
     0xeb, 0x4e, 0x9b, 0x52, 0x2f, 0xd3, 0xdc, 0x4c, 0x41, 0x22, 0x6c, 0xf6, 0x7a, 0xb3, 0x68, 0x59},
    /* SQRT_AD_MINUS_ONE = sqrt(a d - 1) */
    {0x1b, 0x2e, 0x7b, 0x49, 0xa0, 0xf6, 0x97, 0x7e, 0xbd, 0x54, 0x78, 0x1b, 0x0c, 0x8e, 0x9d, 0xaf,
     0xfd, 0xd1, 0xf5, 0x31, 0xc9, 0xfc, 0x3c, 0x0f, 0xac, 0x48, 0x83, 0x2b, 0xbf, 0x31, 0x69, 0x37},
    /* MINUS_ONE */
    {0xec, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
     0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x7f},
    /* MONTGOMERY_A = 486662 */
    {0x06, 0x6d, 0x07},
    /* MONTGOMERY_A_NEG */
    {0xe7, 0x92, 0xf8, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
     0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x7f},
    /* ED25519_SQRTAM2 = sqrt(-A - 2) */
    {0x06, 0x7e, 0x45, 0xff, 0xaa, 0x04, 0x6e, 0xcc, 0x82, 0x1a, 0x7d, 0x4b, 0xd1, 0xd3, 0xa1, 0xc5,
     0x7e, 0x4f, 0xfc, 0x03, 0xdc, 0x08, 0x7b, 0xd2, 0xbb, 0x06, 0xa0, 0x60, 0xf4, 0xed, 0x26, 0x0f},
    /* FE_C2 = 2^((p+3)/8) */
    {0xb1, 0xa0, 0x0e, 0x4a, 0x27, 0x1b, 0xee, 0xc4, 0x78, 0xe4, 0x2f, 0xad, 0x06, 0x18, 0x43, 0x2f,
     0xa7, 0xd7, 0xfb, 0x3d, 0x99, 0x00, 0x4d, 0x2b, 0x0b, 0xdf, 0xc1, 0x4f, 0x80, 0x24, 0x83, 0x2b},
    /* EDWARDS_D */
    {0xa3, 0x78, 0x59, 0x13, 0xca, 0x4d, 0xeb, 0x75, 0xab, 0xd8, 0x41, 0x41, 0x4d, 0x0a, 0x70, 0x00,
     0x98, 0xe8, 0x79, 0x77, 0x79, 0x40, 0xc7, 0x8c, 0x73, 0xfe, 0x6f, 0x2b, 0xee, 0x6c, 0x03, 0x52},
    /* SQRT_M1 */
    {0xb0, 0xa0, 0x0e, 0x4a, 0x27, 0x1b, 0xee, 0xc4, 0x78, 0xe4, 0x2f, 0xad, 0x06, 0x18, 0x43, 0x2f,
     0xa7, 0xd7, 0xfb, 0x3d, 0x99, 0x00, 0x4d, 0x2b, 0x0b, 0xdf, 0xc1, 0x4f, 0x80, 0x24, 0x83, 0x2b},
};

static void K(fe51 *o, int k) { fe_from_bytes(o, KB[k]); }

void h2c_oracle_constant(uint8_t out[32], int k) { memcpy(out, KB[k], 32); }

/* RistrettoPoint::elligator_ristretto_flavor, C/ristretto/elligator.rs:15-51 */
static void elligator_ristretto_flavor(ge_p3 *o, const fe51 *r_0)
{
    fe51 i, d, one_minus_d_sq, d_minus_one_sq, c, one, r, t, N_s, D, s, s_prime, N_t, s_sq, sad;
    K(&i, K_SQRTM1); K(&d, K_D); K(&one_minus_d_sq, K_ONE_MINUS_D_SQ); K(&d_minus_one_sq, K_D_MINUS_ONE_SQ);
    K(&c, K_MINUS_ONE); fe_one(&one);
    fe_square(&t, r_0); fe_mul(&r, &i, &t);                              /* r = i * r_0^2 */
    fe_add(&t, &r, &one); fe_mul(&N_s, &t, &one_minus_d_sq);             /* N_s = (r + 1) * (1 - d^2) */
    fe51 dr, a, b;
    fe_mul(&dr, &d, &r); fe_sub(&a, &c, &dr); fe_add(&b, &r, &d); fe_mul(&D, &a, &b);   /* D = (c - d r) * (r + d) */
    int Ns_D_is_sq = fe_sqrt_ratio_i(&s, &N_s, &D);
    fe_mul(&s_prime, &s, r_0);
    int s_prime_is_pos = !fe_is_negative(&s_prime);
    fe_cond_negate(&s_prime, s_prime_is_pos);
    fe_cond_assign(&s, &s_prime, !Ns_D_is_sq);
    fe_cond_assign(&c, &r, !Ns_D_is_sq);
    fe_sub(&t, &r, &one); fe_mul(&t, &c, &t); fe_mul(&t, &t, &d_minus_one_sq); fe_sub(&N_t, &t, &D);
    fe_square(&s_sq, &s);
    ge_p1p1 W;
    K(&sad, K_SQRT_AD_MINUS_ONE);
    fe_add(&t, &s, &s); fe_mul(&W.X, &t, &D);
    fe_mul(&W.Z, &N_t, &sad);
    fe_sub(&W.Y, &one, &s_sq);
    fe_add(&W.T, &one, &s_sq);
    ge_p1p1_to_p3(o, &W);
}

/* RistrettoPoint::from_uniform_bytes, C/ristretto.rs:774-790 */
static void from_uniform_bytes_point(ge_p3 *o, const uint8_t bytes[64])
{
    fe51 r_1, r_2; ge_p3 R_1, R_2;
    fe_from_bytes(&r_1, bytes); elligator_ristretto_flavor(&R_1, &r_1);
    fe_from_bytes(&r_2, bytes + 32); elligator_ristretto_flavor(&R_2, &r_2);
    ge_p3_add(o, &R_1, &R_2);
}

void h2c_ristretto_elligator(uint8_t out[32], const uint8_t r0[32])
{
    fe51 r; ge_p3 P; fe_from_bytes(&r, r0); elligator_ristretto_flavor(&P, &r); ristretto_compress(out, &P);
}

void h2c_from_uniform_bytes(uint8_t out[32], const uint8_t in[64])
{
    ge_p3 P; from_uniform_bytes_point(&P, in); ristretto_compress(out, &P);
}

/* RistrettoPoint::hash_from_bytes::<Sha512> / from_hash, C/ristretto.rs:736-761 */
void h2c_hash_from_bytes(uint8_t out[32], const uint8_t *msg, size_t len)
{
    uint8_t h[64]; sha512(h, msg, len); h2c_from_uniform_bytes(out, h);
}

/* FieldElement::from_bytes_wide, C/field.rs:110-147 */
void h2c_from_bytes_wide(uint8_t out[32], const uint8_t bytes[64])
{
    uint8_t fl[32], gl[32];
    memcpy(fl, bytes, 32); memcpy(gl, bytes + 32, 32);
    uint16_t fl_top_bit = fl[31] >> 7, gl_top_bit = gl[31] >> 7;
    fl[31] &= 0x7f; gl[31] &= 0x7f;
    fe51 fe_f, fe_g, top, tt, t;
    fe_from_bytes(&fe_f, fl); fe_from_bytes(&fe_g, gl);
    uint16_t addend = fl_top_bit * 19 + gl_top_bit * 722;
    uint8_t ab[32] = {0}; ab[0] = addend & 0xff; ab[1] = addend >> 8;
    fe_from_bytes(&top, ab);
    fe_add(&fe_f, &fe_f, &top);
    uint8_t tb[32] = {38};
    fe_from_bytes(&tt, tb);
    fe_mul(&t, &tt, &fe_g);
    fe_add(&fe_f, &fe_f, &t);
    fe_to_bytes(out, &fe_f);
}

/* expand_msg_xmd::<Sha512>, C/field.rs:440-516; outlen <= 128 */
void h2c_expand_msg_xmd(uint8_t *out, const uint8_t *msg, size_t mlen, const uint8_t *dst, size_t dlen, size_t outlen)
{
    uint8_t z_pad[128] = {0}, l_i_b_str[2] = {(uint8_t)(outlen >> 8), (uint8_t)outlen}, zero = 0, dl = (uint8_t)dlen;
    size_t ell = (outlen + 63) / 64;
    uint8_t b_0[64], buf[128];
    sha512_ctx h;
    sha512_init(&h);
    sha512_update(&h, z_pad, 128); sha512_update(&h, msg, mlen); sha512_update(&h, l_i_b_str, 2);
    sha512_update(&h, &zero, 1); sha512_update(&h, dst, dlen); sha512_update(&h, &dl, 1);
    sha512_final(&h, b_0);
    uint8_t one = 1;
    sha512_init(&h);
    sha512_update(&h, b_0, 64); sha512_update(&h, &one, 1); sha512_update(&h, dst, dlen); sha512_update(&h, &dl, 1);
    sha512_final(&h, buf);
    for (size_t i = 2; i <= ell; i++) {
        uint8_t xor_bs[64], ib = (uint8_t)i;
        for (int k = 0; k < 64; k++) xor_bs[k] = b_0[k] ^ buf[(i - 2) * 64 + k];
        sha512_init(&h);
        sha512_update(&h, xor_bs, 64); sha512_update(&h, &ib, 1); sha512_update(&h, dst, dlen); sha512_update(&h, &dl, 1);
        sha512_final(&h, buf + (i - 1) * 64);
    }
    memcpy(out, buf, outlen);
}

/* FieldElement::hash_to_field::<Sha512, count>, C/field.rs:397-428: count canonical elements */
void h2c_hash_to_field(uint8_t *out, const uint8_t *msg, size_t mlen, const uint8_t *dst, size_t dlen, int count)
{
    uint8_t ub[96];
    h2c_expand_msg_xmd(ub, msg, mlen, dst, dlen, 48 * (size_t)count);
    for (int i = 0; i < count; i++) {
        uint8_t wide[64] = {0};
        for (int k = 0; k < 48; k++) wide[k] = ub[48 * i + 47 - k];
        h2c_from_bytes_wide(out + 32 * i, wide);
    }
}

/* montgomery::elligator_encode, C/montgomery.rs:276-363 */
static void elligator_encode(fe51 *xn_o, fe51 *xd_o, fe51 *y_o, const fe51 *u)
{
    fe51 one, c2, A, x1n, sm1, tv1, xd, tv2, gxd, gx1, tv3, y11, y12, y1, x2n, y21, y22, gx2, y2, xn, y, ny;
    fe_one(&one); K(&c2, K_ELL2_C2); K(&A, K_MONT_A); K(&x1n, K_MONT_A_NEG); K(&sm1, K_SQRTM1);
    fe_square2(&tv1, u);
    fe_add(&xd, &one, &tv1);
    fe_square(&tv2, &xd);
    fe_mul(&gxd, &tv2, &xd);
    fe_mul(&gx1, &A, &tv1);
    fe_mul(&gx1, &gx1, &x1n);
    fe_add(&gx1, &gx1, &tv2);
    fe_mul(&gx1, &gx1, &x1n);
    fe_square(&tv3, &gxd);
    fe_square(&tv2, &tv3);
    fe_mul(&tv3, &tv3, &gxd);
    fe_mul(&tv3, &tv3, &gx1);
    fe_mul(&tv2, &tv2, &tv3);
    fe_pow_p58(&y11, &tv2);
    fe_mul(&y11, &y11, &tv3);
    fe_mul(&y12, &y11, &sm1);
    fe_square(&tv2, &y11); fe_mul(&tv2, &tv2, &gxd);
    int e1 = fe_ct_eq(&tv2, &gx1);
    y1 = y12; fe_cond_assign(&y1, &y11, e1);
    fe_mul(&x2n, &x1n, &tv1);
    fe_mul(&y21, &y11, u);
    fe_mul(&y21, &y21, &c2);
    fe_mul(&y22, &y21, &sm1);
    fe_mul(&gx2, &gx1, &tv1);
    fe_square(&tv2, &y21); fe_mul(&tv2, &tv2, &gxd);
    int e2 = fe_ct_eq(&tv2, &gx2);
    y2 = y22; fe_cond_assign(&y2, &y21, e2);
    fe_square(&tv2, &y1); fe_mul(&tv2, &tv2, &gxd);
    int e3 = fe_ct_eq(&tv2, &gx1);
    xn = x2n; fe_cond_assign(&xn, &x1n, e3);
    y = y2; fe_cond_assign(&y, &y1, e3);
    int e4 = fe_is_negative(&y);
    fe_neg(&ny, &y);
    fe_cond_assign(&y, &ny, e3 ^ e4);
    *xn_o = xn; *xd_o = xd; *y_o = y;
}

/* EdwardsPoint::map_to_curve, C/edwards.rs:651-686 */
static void map_to_curve(ge_p3 *o, const fe51 *u)
{
    fe51 c1, xMn, xMd, yMn, yMd, xn, xd, yn, yd, tv1, zero, one;
    K(&c1, K_SQRTAM2); fe_zero(&zero); fe_one(&one);
    elligator_encode(&xMn, &xMd, &yMn, u); yMd = one;
    fe_mul(&xn, &xMn, &yMd);
    fe_mul(&xn, &xn, &c1);
    fe_mul(&xd, &xMd, &yMn);
    fe_sub(&yn, &xMn, &xMd);
    fe_add(&yd, &xMn, &xMd);
    fe_mul(&tv1, &xd, &yd);
    int e = fe_ct_eq(&tv1, &zero);
    fe_cond_assign(&xn, &zero, e);
    fe_cond_assign(&xd, &one, e);
    fe_cond_assign(&yn, &one, e);
    fe_cond_assign(&yd, &one, e);
    fe_mul(&o->X, &xn, &yd);
    fe_mul(&o->Y, &xd, &yn);
    fe_mul(&o->Z, &xd, &yd);
    fe_mul(&o->T, &xn, &yn);
}

void h2c_map_to_curve(uint8_t out[32], const uint8_t u_bytes[32])
{
    fe51 u; ge_p3 P; fe_from_bytes(&u, u_bytes); map_to_curve(&P, &u); ge_compress(out, &P);
}

/* EdwardsPoint::hash_to_curve (count 2, C/edwards.rs:736-750) / encode_to_curve (count 1, :710-721) with Sha512 */
void h2c_hash_to_curve(uint8_t out[32], const uint8_t *msg, size_t mlen, const uint8_t *dst, size_t dlen, int count)
{
    uint8_t fb[64];
    h2c_hash_to_field(fb, msg, mlen, dst, dlen, count);
    fe51 u; ge_p3 Q, R;
    fe_from_bytes(&u, fb); map_to_curve(&Q, &u);
    if (count == 2) {
        ge_p3 Q1; fe_from_bytes(&u, fb + 32); map_to_curve(&Q1, &u);
        ge_p3_add(&R, &Q, &Q1);
    } else {
        R = Q;
    }
    ge_mul_by_pow_2(&Q, &R, 3);                                          /* mul_by_cofactor, C/edwards.rs:1393-1395 */
    ge_compress(out, &Q);
}

/* batches over the flat message layout (message i = msgs[offs[i] .. offs[i+1])); kind 0: hash_from_bytes,
 * 1: encode_to_curve, 2: hash_to_curve */
void h2c_flat_batch(uint8_t *out, const uint8_t *msgs, const uint64_t *offs, size_t n, const uint8_t *dst, size_t dlen,
                    int kind)
{
    for (size_t i = 0; i < n; i++) {
        const uint8_t *m = msgs + offs[i];
        size_t len = (size_t)(offs[i + 1] - offs[i]);
        if (kind == 0) h2c_hash_from_bytes(out + 32 * i, m, len);
        else h2c_hash_to_curve(out + 32 * i, m, len, dst, dlen, kind);
    }
}

void h2c_from_uniform_batch(uint8_t *out, const uint8_t *in, size_t n)
{
    for (size_t i = 0; i < n; i++) h2c_from_uniform_bytes(out + 32 * i, in + 64 * i);
}
