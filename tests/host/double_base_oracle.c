/*
 * double_base_oracle.c -- CPU oracle of the batched variable-time double-base scalar multiplication a A + b B, B the
 * Ed25519 basepoint.  TEST INFRASTRUCTURE ONLY (compiled together with the oracle library's C sources by
 * tests/double_base_oracle.py): the parity source of the GPU double-base batch and the CPU baseline of
 * tools/bench_double_base.py.
 *
 * dbo_vartime_double_base_naf restates the algorithm of C/backend/serial/scalar_mul/vartime_double_base.rs:23-72 step
 * by step: a width-5 NAF of a over the NafLookupTable5 [A, 3A, .., 15A] of projective Niels points, a width-8 NAF of b
 * over the 64 affine Niels odd multiples [B, 3B, .., 127B] (the precomputed-tables branch, constants
 * AFFINE_ODD_MULTIPLES_OF_BASEPOINT), the search for the highest non-zero digit and the double-and-add loop on projective
 * points.  The oracle library's own edwards_vartime_double_scalar_mul_basepoint computes the same value through the
 * vartime Straus over [A, B]; both are exposed so that the tests can hold them against each other.
 */
#include "oracle.h"
#include "constants.h"
#include <pthread.h>
#include <string.h>

enum { FMT_COMPRESSED = 0, FMT_EXTENDED = 1, FMT_RISTRETTO = 2 };

/* EdwardsPoint::as_affine_niels, C/edwards.rs:551-561 */
static void to_aniels(ge_aniels *o, const ge_p3 *p)
{
    fe51 recip, x, y, d2;
    memcpy(d2.v, K_EDWARDS_D2, sizeof d2.v);
    fe_invert(&recip, &p->Z);
    fe_mul(&x, &p->X, &recip);
    fe_mul(&y, &p->Y, &recip);
    fe_add(&o->y_plus_x, &y, &x);
    fe_sub(&o->y_minus_x, &y, &x);
    fe_mul(&o->xy2d, &x, &y); fe_mul(&o->xy2d, &o->xy2d, &d2);
}

/* NafLookupTable8<AffineNielsPoint>::from (C/window.rs:266-276): [P, 3P, 5P, ..., 127P] */
typedef struct { ge_aniels t[64]; } naf_table8;
static void naf_table8_from(naf_table8 *t, const ge_p3 *p)
{
    ge_p3 p2;
    to_aniels(&t->t[0], p);
    ge_p3_double(&p2, p);
    for (int i = 0; i < 63; i++) {
        ge_p1p1 r; ge_p3 e;
        ge_add_aniels(&r, &p2, &t->t[i]); ge_p1p1_to_p3(&e, &r); to_aniels(&t->t[i + 1], &e);
    }
}

static naf_table8 g_table_B;
static pthread_once_t g_table_once = PTHREAD_ONCE_INIT;
static void table_B_init(void)
{
    ge_p3 B; ge_basepoint(&B);
    naf_table8_from(&g_table_B, &B);
}

/* vartime_double_base.rs:23-72 */
void dbo_vartime_double_base_naf(ge_p3 *o, const uint8_t a[32], const ge_p3 *A, const uint8_t b[32])
{
    int8_t a_naf[256], b_naf[256];
    scalar_non_adjacent_form(a_naf, a, 5);                          /* :24 */
    scalar_non_adjacent_form(b_naf, b, 8);                          /* :27-30 (precomputed tables) */
    int i = 255;                                                    /* :37-43, find the starting index */
    for (int j = 255; j >= 0; j--) {
        i = j;
        if (a_naf[i] != 0 || b_naf[i] != 0) break;
    }
    ge_naf_table5 table_A;                                          /* :45 */
    ge_naf_table5_from(&table_A, A);
    pthread_once(&g_table_once, table_B_init);                      /* :47-48 */
    const naf_table8 *table_B = &g_table_B;
    ge_p2 r; ge_p2_identity(&r);                                    /* :52 */
    for (;;) {                                                      /* :53-69 */
        ge_p1p1 t; ge_p3 e;
        ge_p2_double(&t, &r);
        if (a_naf[i] > 0) { ge_p1p1_to_p3(&e, &t); ge_add_pniels(&t, &e, &table_A.t[a_naf[i] / 2]); }
        else if (a_naf[i] < 0) { ge_p1p1_to_p3(&e, &t); ge_sub_pniels(&t, &e, &table_A.t[-a_naf[i] / 2]); }
        if (b_naf[i] > 0) { ge_p1p1_to_p3(&e, &t); ge_add_aniels(&t, &e, &table_B->t[b_naf[i] / 2]); }
        else if (b_naf[i] < 0) { ge_p1p1_to_p3(&e, &t); ge_sub_aniels(&t, &e, &table_B->t[-b_naf[i] / 2]); }
        ge_p1p1_to_p2(&r, &t);
        if (i == 0) break;
        i -= 1;
    }
    ge_p2_to_p3(o, &r);                                             /* :71 */
}

static int load_point(ge_p3 *p, const uint8_t *in, int fmt)
{
    if (fmt == FMT_EXTENDED) {
        uint64_t l[20];
        memcpy(l, in, 160);
        ge_p3_from_limbs(p, l);
        return 1;
    }
    return fmt == FMT_RISTRETTO ? ristretto_decompress(p, in) : ge_decompress(p, in);
}

/* one item in the format of the C ABI; naf = 0: the oracle library's Straus-based value.  Returns 1 if A decodes (else
 * out = the identity's encoding). */
int dbo_one(uint8_t out[32], const uint8_t ab[64], const uint8_t *point, int fmt, int naf)
{
    ge_p3 A, R;
    const int good = load_point(&A, point, fmt);
    if (!good) ge_identity(&R);
    else if (naf) dbo_vartime_double_base_naf(&R, ab, &A, ab + 32);
    else edwards_vartime_double_scalar_mul_basepoint(&R, ab, &A, ab + 32);
    if (fmt == FMT_RISTRETTO) ristretto_compress(out, &R);
    else ge_compress(out, &R);
    return good;
}

typedef struct {
    uint8_t *out, *ok;
    const uint8_t *ab, *points;
    int fmt;
    size_t lo, hi;
} dbo_job;

static void *dbo_run(void *arg)
{
    const dbo_job *j = (const dbo_job *)arg;
    const size_t pin = j->fmt == FMT_EXTENDED ? 160 : 32;
    for (size_t i = j->lo; i < j->hi; i++) {
        const int good = dbo_one(j->out + 32 * i, j->ab + 64 * i, j->points + pin * i, j->fmt, 1);
        if (j->ok) j->ok[i] = (uint8_t)good;
    }
    return NULL;
}

/* n items over `threads` threads (1: the calling thread), each by the faithful NAF algorithm.  Returns 1 if some point
 * does not decode (DALEK_NONE), else 0. */
int dbo_batch(uint8_t *out, uint8_t *ok, const uint8_t *ab, const uint8_t *points, int fmt, size_t n, int threads)
{
    enum { MAX_THREADS = 256 };
    if (threads < 1) threads = 1;
    if (threads > MAX_THREADS) threads = MAX_THREADS;
    pthread_once(&g_table_once, table_B_init);
    dbo_job jobs[MAX_THREADS];
    pthread_t tid[MAX_THREADS];
    for (int t = 0; t < threads; t++) {
        jobs[t] = (dbo_job){out, ok, ab, points, fmt, n * t / threads, n * (t + 1) / threads};
        if (t) pthread_create(&tid[t], NULL, dbo_run, &jobs[t]);
    }
    dbo_run(&jobs[0]);
    for (int t = 1; t < threads; t++) pthread_join(tid[t], NULL);
    if (ok)
        for (size_t i = 0; i < n; i++) if (!ok[i]) return 1;
    return 0;
}
