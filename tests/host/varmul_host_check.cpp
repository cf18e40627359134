// Host build of the device variable-base scalar multiplication (varmul.cuh over fe64.cuh / ge64.cuh) with the
// operand-scale assertions of fe64.cuh and the limb-bound assertions of fe.cuh enabled, exported with a tiny C ABI for
// tests/test_varmul_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the multiplication the kernels run keeps every
// fe64_mul / fe64_sq operand within the scale rule and gives the reference's bytes.  Decoding and encoding use the same
// ge.cuh functions as the kernels (csrc/varmul.cu).
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/varmul.cuh"
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

extern "C" {
// out = encode(s P); clamp: clamp_integer first.  Returns 1 if P decodes (else out = the identity's encoding).
int h_mul(uint8_t *out, const uint8_t *scalar, const uint8_t *point, int fmt, int clamp)
{
    uint32_t s[8];
    memcpy(s, scalar, 32);
    if (clamp) x25519_clamp(s);
    ge_p3 p;
    const uint32_t good = load_point(p, point, fmt);
    ge64_p3 P, Q;
    ge64_from_p3(P, p);
    VarmulLocalTab tab;
    varmul(Q, s, P, tab);
    ge_p3 q;
    ge64_to_p3(q, Q);
    uint32_t w[8];
    if (fmt == 2) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
    memcpy(out, w, 32);
    return (int)good;
}

// is_small_order | is_torsion_free << 1 | decoded << 2, or 0 for an undecodable point (fmt 0 or 1)
int h_torsion(const uint8_t *point, int fmt)
{
    ge_p3 p;
    if (!load_point(p, point, fmt)) return 0;
    ge64_p3 P;
    ge64_from_p3(P, p);
    VarmulLocalTab tab;
    return (int)(varmul_torsion_flags(P, tab) | 4u);
}
}
