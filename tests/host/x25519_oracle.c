/* x25519_oracle.c -- CPU oracle for X25519, restated in plain C from x25519-dalek and curve25519-dalek's montgomery.rs.
 * TEST INFRASTRUCTURE: the byte-for-byte parity source of the GPU X25519 paths and their one-core CPU baseline
 * (tests/x25519_oracle.py loads it).  It shares no code with the engine: its own radix-2^51 field over unsigned
 * __int128 products, and inversion by square-and-multiply over the bits of p - 2.
 *   clamp_integer               C/scalar.rs:1407-1412
 *   MontgomeryPoint::mul_bits_be C/montgomery.rs:183-211   (Costello-Smith algorithm 8)
 *   differential_add_and_double C/montgomery.rs:430-468
 *   ProjectivePoint::as_affine  C/montgomery.rs:409-412    (W = 0 gives u = 0)
 *   x25519                      x25519-dalek x25519.rs:390-392 (mul_clamped, C/montgomery.rs:150-161)
 *   EdwardsPoint::to_montgomery C/edwards.rs:580-590       (u = (Z + Y) / (Z - Y); the identity gives 0) */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t v[5]; } fe;          /* radix 2^51, limbs < 2^52 between operations */

#define MASK51 ((1ULL << 51) - 1)

static void fe_set(fe *h, uint64_t x) { memset(h, 0, sizeof *h); h->v[0] = x; }

/* FieldElement::from_bytes: little endian, bit 255 ignored, no reduction */
static void fe_load(fe *h, const uint8_t s[32])
{
    uint64_t w[4];
    for (int i = 0; i < 4; i++) {
        w[i] = 0;
        for (int b = 7; b >= 0; b--) w[i] = (w[i] << 8) | s[8 * i + b];
    }
    h->v[0] = w[0] & MASK51;
    h->v[1] = ((w[0] >> 51) | (w[1] << 13)) & MASK51;
    h->v[2] = ((w[1] >> 38) | (w[2] << 26)) & MASK51;
    h->v[3] = ((w[2] >> 25) | (w[3] << 39)) & MASK51;
    h->v[4] = (w[3] >> 12) & MASK51;
}

static void fe_reduce_weak(fe *h)
{
    uint64_t c;
    for (int i = 0; i < 4; i++) { c = h->v[i] >> 51; h->v[i] &= MASK51; h->v[i + 1] += c; }
    c = h->v[4] >> 51; h->v[4] &= MASK51; h->v[0] += 19 * c;
    c = h->v[0] >> 51; h->v[0] &= MASK51; h->v[1] += c;
}

static void fe_add(fe *h, const fe *a, const fe *b)
{
    for (int i = 0; i < 5; i++) h->v[i] = a->v[i] + b->v[i];
    fe_reduce_weak(h);
}

/* a - b + 4p, limb-wise non-negative for limbs < 2^53 */
static void fe_sub(fe *h, const fe *a, const fe *b)
{
    h->v[0] = a->v[0] + 4 * ((1ULL << 51) - 19) - b->v[0];
    for (int i = 1; i < 5; i++) h->v[i] = a->v[i] + 4 * MASK51 - b->v[i];
    fe_reduce_weak(h);
}

static void fe_mul(fe *h, const fe *a, const fe *b)
{
    u128 t[5] = {0, 0, 0, 0, 0};
    for (int i = 0; i < 5; i++)
        for (int j = 0; j < 5; j++) {
            u128 p = (u128)a->v[i] * b->v[j];
            if (i + j < 5) t[i + j] += p; else t[i + j - 5] += p * 19;
        }
    uint64_t r[5], c = 0;                      /* c < 2^61 */
    for (int i = 0; i < 5; i++) { t[i] += c; r[i] = (uint64_t)t[i] & MASK51; c = (uint64_t)(t[i] >> 51); }
    u128 x = (u128)r[0] + (u128)c * 19;
    r[0] = (uint64_t)x & MASK51;
    r[1] += (uint64_t)(x >> 51);
    for (int i = 0; i < 5; i++) h->v[i] = r[i];
    fe_reduce_weak(h);
}

static void fe_sq(fe *h, const fe *a) { fe_mul(h, a, a); }

/* a^(p-2) = a^(2^255 - 21) by left-to-right square-and-multiply; 0 -> 0 */
static void fe_invert(fe *h, const fe *a)
{
    /* p - 2 = 2^255 - 21: bits 254..5 set, then bits 4..0 = 01011 */
    fe r; fe_set(&r, 1);
    for (int i = 254; i >= 0; i--) {
        int bit = i >= 5 ? 1 : ((0x0b >> i) & 1);
        fe_sq(&r, &r);
        if (bit) fe_mul(&r, &r, a);
    }
    *h = r;
}

/* FieldElement::to_bytes: fully reduced, little endian */
static void fe_store(uint8_t s[32], const fe *f)
{
    fe h = *f;
    fe_reduce_weak(&h);
    fe_reduce_weak(&h);
    /* h < 2^255 + small; subtract p if h >= p */
    uint64_t q = (h.v[0] + 19) >> 51;
    for (int i = 1; i < 5; i++) q = (h.v[i] + q) >> 51;
    h.v[0] += 19 * q;
    uint64_t c;
    for (int i = 0; i < 4; i++) { c = h.v[i] >> 51; h.v[i] &= MASK51; h.v[i + 1] += c; }
    h.v[4] &= MASK51;
    uint64_t w[4];
    w[0] = h.v[0] | (h.v[1] << 51);
    w[1] = (h.v[1] >> 13) | (h.v[2] << 38);
    w[2] = (h.v[2] >> 26) | (h.v[3] << 25);
    w[3] = (h.v[3] >> 39) | (h.v[4] << 12);
    for (int i = 0; i < 4; i++)
        for (int b = 0; b < 8; b++) s[8 * i + b] = (uint8_t)(w[i] >> (8 * b));
}

static void fe_cswap(fe *a, fe *b, uint64_t c)
{
    uint64_t m = 0 - c;
    for (int i = 0; i < 5; i++) { uint64_t t = m & (a->v[i] ^ b->v[i]); a->v[i] ^= t; b->v[i] ^= t; }
}

void x25519_clamp_integer(uint8_t out[32], const uint8_t in[32])
{
    memcpy(out, in, 32);
    out[0] &= 0xf8;
    out[31] &= 0x7f;
    out[31] |= 0x40;
}

typedef struct { fe U, W; } mont_pt;

static void differential_add_and_double(mont_pt *P, mont_pt *Q, const fe *u_pmq)
{
    fe t0, t1, t2, t3, t4, t5, t6, t7, t8, t9, t10, t11, t12, t13, t14, t15, t16, t17, a24;
    fe_set(&a24, 121666);
    fe_add(&t0, &P->U, &P->W);
    fe_sub(&t1, &P->U, &P->W);
    fe_add(&t2, &Q->U, &Q->W);
    fe_sub(&t3, &Q->U, &Q->W);
    fe_sq(&t4, &t0);
    fe_sq(&t5, &t1);
    fe_sub(&t6, &t4, &t5);
    fe_mul(&t7, &t0, &t3);
    fe_mul(&t8, &t1, &t2);
    fe_add(&t9, &t7, &t8);
    fe_sub(&t10, &t7, &t8);
    fe_sq(&t11, &t9);
    fe_sq(&t12, &t10);
    fe_mul(&t13, &a24, &t6);
    fe_mul(&t14, &t4, &t5);
    fe_add(&t15, &t13, &t5);
    fe_mul(&t16, &t6, &t15);
    fe_mul(&t17, u_pmq, &t12);
    P->U = t14; P->W = t16;
    Q->U = t11; Q->W = t17;
}

/* u([n] P) for u = u(P) and n given by its `nbits` low bits, processed from bit nbits-1 down to bit 0 */
void x25519_mul_bits_be(uint8_t out[32], const uint8_t u_bytes[32], const uint8_t scalar[32], unsigned nbits)
{
    fe u; fe_load(&u, u_bytes);
    mont_pt x0, x1;
    fe_set(&x0.U, 1); fe_set(&x0.W, 0);
    x1.U = u; fe_set(&x1.W, 1);
    uint64_t prev = 0;
    for (int i = (int)nbits - 1; i >= 0; i--) {
        uint64_t bit = (scalar[i >> 3] >> (i & 7)) & 1;
        uint64_t choice = prev ^ bit;
        fe_cswap(&x0.U, &x1.U, choice); fe_cswap(&x0.W, &x1.W, choice);
        differential_add_and_double(&x0, &x1, &u);
        prev = bit;
    }
    fe_cswap(&x0.U, &x1.U, prev); fe_cswap(&x0.W, &x1.W, prev);
    fe wi, r;
    fe_invert(&wi, &x0.W);
    fe_mul(&r, &x0.U, &wi);
    fe_store(out, &r);
}

/* x25519(k, u): Scalar * MontgomeryPoint runs mul_bits_be over bits 254..0 of the clamped k */
void x25519_scalarmult(uint8_t out[32], const uint8_t k[32], const uint8_t u[32])
{
    uint8_t c[32];
    x25519_clamp_integer(c, k);
    x25519_mul_bits_be(out, u, c, 255);
}

void x25519_scalarmult_batch(uint8_t *out, const uint8_t *k, const uint8_t *u, size_t n)
{
    for (size_t i = 0; i < n; i++) x25519_scalarmult(out + 32 * i, k + 32 * i, u + 32 * i);
}

/* EdwardsPoint::to_montgomery on the reference's in-memory point (20 u64 radix-2^51 limbs X | Y | Z | T, limbs < 2^54) */
void x25519_edwards_to_montgomery(uint8_t out[32], const uint64_t limbs[20])
{
    fe Y, Z, num, den, inv, u;
    for (int i = 0; i < 5; i++) { Y.v[i] = limbs[5 + i]; Z.v[i] = limbs[10 + i]; }
    fe_reduce_weak(&Y); fe_reduce_weak(&Z);
    fe_add(&num, &Z, &Y);
    fe_sub(&den, &Z, &Y);
    fe_invert(&inv, &den);
    fe_mul(&u, &num, &inv);
    fe_store(out, &u);
}
