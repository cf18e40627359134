/*
 * montgomery_oracle.c -- CPU oracle of the MontgomeryPoint operations of curve25519-dalek's montgomery.rs.  TEST
 * INFRASTRUCTURE ONLY (compiled together with the oracle library's C sources by tests/montgomery_oracle.py): the parity
 * source of the GPU MontgomeryPoint batches and of the constant-time fixed-base batch.  It uses the oracle library's
 * field (the reference's serial u64 backend), decompression, compression and scalar multiplication, and no engine code.
 *
 *   MontgomeryPoint::mul_bits_be  C/montgomery.rs:176-211   Costello-Smith algorithm 8 over any number of bits
 *                                                           (here up to 512), differential_add_and_double :430-468,
 *                                                           as_affine :409-412
 *   Scalar * MontgomeryPoint      C/montgomery.rs:484-492   mul_bits_be over bits 254..0 of the Scalar
 *   MontgomeryPoint::to_edwards   C/montgomery.rs:223-268   u == -1 -> None; y = (u-1)/(u+1); y[31] ^= sign << 7 (u8);
 *                                                           CompressedEdwardsY::decompress
 *   EdwardsPoint::mul_base(s) -> compress / RistrettoPoint compress / to_montgomery (C/edwards.rs:580-590): the value
 *                                                           s B of ge_scalarmul, any s < 2^255
 */
#include "oracle.h"
#include <pthread.h>
#include <string.h>
#include <unistd.h>

enum { FMT_COMPRESSED = 0, FMT_RISTRETTO = 2, FMT_MONTGOMERY = 3 };

static void fe_small(fe51 *o, uint64_t x) { fe_zero(o); o->v[0] = x; }

/* ProjectivePoint::conditional_swap */
static void fe_cswap(fe51 *a, fe51 *b, int c)
{
    fe51 t = *a;
    fe_cond_assign(a, b, c);
    fe_cond_assign(b, &t, c);
}

/* differential_add_and_double (C/montgomery.rs:430-468), step by step */
static void differential_add_and_double(fe51 *PU, fe51 *PW, fe51 *QU, fe51 *QW, const fe51 *affine_PmQ)
{
    fe51 t0, t1, t2, t3, t4, t5, t6, t7, t8, t9, t10, t11, t12, t13, t14, t15, t16, t17, t18, a24;
    fe_small(&a24, 121666);                         /* APLUS2_OVER_FOUR */
    fe_add(&t0, PU, PW);
    fe_sub(&t1, PU, PW);
    fe_add(&t2, QU, QW);
    fe_sub(&t3, QU, QW);
    fe_square(&t4, &t0);
    fe_square(&t5, &t1);
    fe_sub(&t6, &t4, &t5);
    fe_mul(&t7, &t0, &t3);
    fe_mul(&t8, &t1, &t2);
    fe_add(&t9, &t7, &t8);
    fe_sub(&t10, &t7, &t8);
    fe_square(&t11, &t9);
    fe_square(&t12, &t10);
    fe_mul(&t13, &a24, &t6);
    fe_mul(&t14, &t4, &t5);
    fe_add(&t15, &t13, &t5);
    fe_mul(&t16, &t6, &t15);
    fe_mul(&t17, affine_PmQ, &t12);
    t18 = t11;
    *PU = t14; *PW = t16;
    *QU = t18; *QW = t17;
}

/* u([b] P) for b = bits nbits-1..0 of the int_bytes-byte little-endian integer `ints` */
void mo_mul_bits_be(uint8_t out[32], const uint8_t u_bytes[32], const uint8_t *ints, unsigned int_bytes, unsigned nbits)
{
    fe51 u, x0U, x0W, x1U, x1W, wi, r;
    fe_from_bytes(&u, u_bytes);
    fe_one(&x0U); fe_zero(&x0W);                    /* ProjectivePoint::identity */
    x1U = u; fe_one(&x1W);
    int prev = 0;
    for (int i = (int)nbits - 1; i >= 0; i--) {
        int bit = (unsigned)i < 8 * int_bytes ? (ints[i >> 3] >> (i & 7)) & 1 : 0;
        int choice = prev ^ bit;
        fe_cswap(&x0U, &x1U, choice); fe_cswap(&x0W, &x1W, choice);
        differential_add_and_double(&x0U, &x0W, &x1U, &x1W, &u);
        prev = bit;
    }
    fe_cswap(&x0U, &x1U, prev); fe_cswap(&x0W, &x1W, prev);
    fe_invert(&wi, &x0W);                           /* as_affine: U * W^(p-2) */
    fe_mul(&r, &x0U, &wi);
    fe_to_bytes(out, &r);
}

/* to_edwards(u, sign) as CompressedEdwardsY; returns 0 for None (out = the identity's encoding) */
int mo_to_edwards(uint8_t out[32], const uint8_t u_bytes[32], uint8_t sign)
{
    fe51 u, one, minus_one, num, den, inv, y;
    uint8_t y_bytes[32];
    ge_p3 P;
    memset(out, 0, 32); out[0] = 1;
    fe_from_bytes(&u, u_bytes);
    fe_one(&one);
    fe_neg(&minus_one, &one);
    if (fe_ct_eq(&u, &minus_one)) return 0;
    fe_sub(&num, &u, &one);
    fe_add(&den, &u, &one);
    fe_invert(&inv, &den);
    fe_mul(&y, &num, &inv);
    fe_to_bytes(y_bytes, &y);
    y_bytes[31] ^= (uint8_t)(sign << 7);
    if (!ge_decompress(&P, y_bytes)) return 0;
    ge_compress(out, &P);
    return 1;
}

/* s B (s < 2^255; clamped first when clamp) encoded as fmt */
void mo_mul_base(uint8_t out[32], const uint8_t s_in[32], int fmt, int clamp)
{
    uint8_t s[32];
    ge_p3 B, P;
    memcpy(s, s_in, 32);
    if (clamp) { s[0] &= 0xf8; s[31] &= 0x7f; s[31] |= 0x40; }    /* clamp_integer, C/scalar.rs:1407-1412 */
    ge_basepoint(&B);
    ge_scalarmul(&P, s, &B);
    if (fmt == FMT_RISTRETTO) ristretto_compress(out, &P);
    else if (fmt == FMT_MONTGOMERY) {                               /* EdwardsPoint::to_montgomery, C/edwards.rs:580-590 */
        fe51 num, den, inv, u;
        fe_add(&num, &P.Z, &P.Y);
        fe_sub(&den, &P.Z, &P.Y);
        fe_invert(&inv, &den);
        fe_mul(&u, &num, &inv);
        fe_to_bytes(out, &u);
    } else ge_compress(out, &P);
}

/* ---- batches over threads: item i of a broadcast input (step 0) is item 0 ---- */
enum { OP_BITS = 0, OP_TO_EDWARDS = 1, OP_MUL_BASE = 2 };

typedef struct {
    int op;
    uint8_t *out, *ok;
    const uint8_t *a, *b;
    size_t a_step, b_step;
    unsigned int_bytes, nbits;
    int fmt, clamp;
    size_t lo, hi;
} job;

static void *run_job(void *arg)
{
    job *j = (job *)arg;
    for (size_t i = j->lo; i < j->hi; i++) {
        if (j->op == OP_BITS) mo_mul_bits_be(j->out + 32 * i, j->b + j->b_step * i, j->a + j->a_step * i, j->int_bytes, j->nbits);
        else if (j->op == OP_TO_EDWARDS) j->ok[i] = (uint8_t)mo_to_edwards(j->out + 32 * i, j->a + 32 * i, j->b[i]);
        else mo_mul_base(j->out + 32 * i, j->a + 32 * i, j->fmt, j->clamp);
    }
    return NULL;
}

static void run_batch(const job *proto, size_t n)
{
    long ncpu = sysconf(_SC_NPROCESSORS_ONLN);
    size_t t = ncpu < 1 ? 1 : (size_t)(ncpu > 32 ? 32 : ncpu);
    if (t > n) t = n ? n : 1;
    pthread_t th[32];
    job jobs[32];
    for (size_t k = 0; k < t; k++) {
        jobs[k] = *proto;
        jobs[k].lo = n * k / t;
        jobs[k].hi = n * (k + 1) / t;
        if (k + 1 < t) pthread_create(&th[k], NULL, run_job, &jobs[k]);
    }
    run_job(&jobs[t - 1]);
    for (size_t k = 0; k + 1 < t; k++) pthread_join(th[k], NULL);
}

/* ints: n_ints (1 or n) integers of int_bytes bytes; us: n_points (1 or n) u coordinates */
void mo_mul_bits_be_batch(uint8_t *out, const uint8_t *ints, unsigned int_bytes, size_t n_ints, unsigned nbits, const uint8_t *us,
                          size_t n_points, size_t n)
{
    job j = {OP_BITS, out, NULL, ints, us, n_ints == 1 ? 0 : int_bytes, n_points == 1 ? 0 : 32, int_bytes, nbits, 0, 0, 0, 0};
    run_batch(&j, n);
}

/* returns the number of None items */
size_t mo_to_edwards_batch(uint8_t *out, uint8_t *ok, const uint8_t *us, const uint8_t *signs, size_t n)
{
    job j = {OP_TO_EDWARDS, out, ok, us, signs, 32, 1, 0, 0, 0, 0, 0, 0};
    run_batch(&j, n);
    size_t none = 0;
    for (size_t i = 0; i < n; i++) none += !ok[i];
    return none;
}

void mo_mul_base_batch(uint8_t *out, const uint8_t *scalars, size_t n, int fmt, int clamp)
{
    job j = {OP_MUL_BASE, out, NULL, scalars, NULL, 32, 0, 0, 0, fmt, clamp, 0, 0};
    run_batch(&j, n);
}
