// Host build of the device double-base scalar multiplication (double_base.cuh over fe64.cuh / ge64.cuh) with the
// operand-scale assertions of fe64.cuh and the limb-bound assertions of fe.cuh enabled, exported with a tiny C ABI for
// tests/test_double_base_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the evaluation the kernels run keeps every
// fe64_mul / fe64_sq operand within the scale rule and gives the reference's bytes.  B's table is staged from the same
// packed affine Niels entries as row 0 of the device's fixed-base table (base.cu), decoding and encoding use the same
// ge.cuh functions as the kernels (csrc/double_base.cu).
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/double_base.cuh"
#include <string.h>

// fmt: 0 CompressedEdwardsY, 1 extended radix-2^51 limbs (160 B), 2 CompressedRistretto; 1 if the point decodes
static uint32_t load_point(ge_p3 &p, const uint8_t *in, int fmt)
{
    if (fmt == 1) {
        uint64_t l[20];
        memcpy(l, in, 160);
        fe_from_limbs51(p.X, l); fe_from_limbs51(p.Y, l + 5); fe_from_limbs51(p.Z, l + 10); fe_from_limbs51(p.T, l + 15);
        return 1;
    }
    uint32_t s[8];
    memcpy(s, in, 32);
    uint32_t good;
    if (fmt == 2) {
        good = ristretto_decompress<1>(p, s);
    } else {
        good = ge_decompress_affine<1>(p.X, p.Y, s);
        fe_1(p.Z);
        fe_mul(p.T, p.X, p.Y);
    }
    if (!good) ge_p3_identity(p);
    return good;
}

// (j+1) B, j = 0..7, as packed affine Niels points and then as the 8 x 15 doubles of the kernels' shared table
static void stage_B(double s_B[8 * 15])
{
    ge_p3 B, P;
    ge_p3_basepoint(B);
    ge_niels nb; ge_affine_to_niels(nb, B.X, B.Y);
    P = B;
    for (int j = 0; j < 8; j++) {
        if (j) ge_madd(P, P, nb, 0);
        fe zi, x, y;
        fe_invert(zi, P.Z);
        fe_mul(x, P.X, zi); fe_mul(y, P.Y, zi);
        ge_niels n; ge_affine_to_niels(n, x, y);
        ge_niels_packed pk; ge_niels_pack(pk, n);
        double_base_stage_B(s_B + 15 * j, pk);
    }
}

extern "C" {
// out = encode(a P + b B), ab = a || b (bit 255 clear).  Returns 1 if P decodes (else out = the identity's encoding).
int h_double_base(uint8_t *out, const uint8_t *ab, const uint8_t *point, int fmt)
{
    static double s_B[8 * 15];
    static int staged = 0;
    if (!staged) { stage_B(s_B); staged = 1; }
    uint32_t a[8], b[8];
    memcpy(a, ab, 32);
    memcpy(b, ab + 32, 32);
    ge_p3 p;
    const uint32_t good = load_point(p, point, fmt);
    ge64_p3 Q;
    DoubleBaseLocal loc;
    double_base_eval(Q, p, a, b, s_B, loc);
    if (!good) ge64_identity(Q);
    ge_p3 q;
    ge64_to_p3(q, Q);
    uint32_t w[8];
    if (fmt == 2) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
    memcpy(out, w, 32);
    return (int)good;
}
}
