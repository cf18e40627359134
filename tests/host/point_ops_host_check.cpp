// Host build of the group operations (point_ops.cuh over ge.cuh / ge64.cuh) with the limb-bound assertions of fe.cuh and
// the operand-scale assertions of fe64.cuh enabled, exported with a tiny C ABI for tests/test_point_ops_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the arithmetic the kernels run (csrc/point_ops.cu)
// keeps every operand within its bound and gives the reference's bytes, and it exposes the sum's chunk plan.
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/point_ops.cuh"
#include <string.h>

// fmt: 0 CompressedEdwardsY, 1 extended radix-2^51 limbs (160 B), 2 CompressedRistretto; 1 if the point decodes (the
// kernels' varmul_load_point, point_load.cuh)
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
    point_cmov_identity(p, 1u - good);
    return good;
}

// enc: 0 CompressedEdwardsY (32 B), 1 CompressedRistretto (32 B), 2 canonical limbs (160 B)
static void encode(uint8_t *out, const ge_p3 &q, int enc)
{
    if (enc == 2) {
        uint64_t l[20];
        point_to_limbs(l, q);
        memcpy(out, l, 160);
        return;
    }
    uint32_t w[8];
    if (enc == 1) ristretto_compress<1>(w, q);
    else ge_compress<1>(w, q);
    memcpy(out, w, 32);
}

extern "C" {
// out = op(A, B) (PO_*), the identity if an input does not decode; returns 1 if both decode (b is read by add / sub only)
int h_op(uint8_t *out, const uint8_t *a, const uint8_t *b, int fmt, int op, int enc)
{
    ge_p3 A, B, R;
    uint32_t good = load_point(A, a, fmt);
    ge_p3_identity(B);
    if (op <= PO_SUB) good &= load_point(B, b, fmt);
    point_apply(R, A, B, op);
    point_cmov_identity(R, 1u - good);
    encode(out, R, enc);
    return (int)good;
}

// eq | both_decoded << 1; b = NULL: the identity
int h_eq(const uint8_t *a, const uint8_t *b, int fmt, int rist)
{
    ge_p3 A, B;
    uint32_t good = load_point(A, a, fmt);
    ge_p3_identity(B);
    if (b) good &= load_point(B, b, fmt);
    const uint32_t e = rist ? ristretto_eq(A, B) : edwards_eq(A, B);
    return (int)((e & good) | (good << 1));
}

// the sum of n points on the FP64 field as the kernels form it: runs of `threads` strided points, then a pairwise tree;
// returns 1 if every point decodes (else out is the identity)
int h_sum(uint8_t *out, const uint8_t *pts, size_t n, int fmt, int threads, int enc)
{
    const size_t sz = fmt == 1 ? 160 : 32;
    fe64 d2;
    { fe k; fe_const_2d(k); fe64_from_fe(d2, k); }
    std::vector<ge64_p3> acc((size_t)threads);
    uint32_t good = 1;
    for (int t = 0; t < threads; t++) {
        ge64_identity(acc[t]);
        for (size_t i = (size_t)t; i < n; i += (size_t)threads) {
            ge_p3 p;
            good &= load_point(p, pts + sz * i, fmt);
            ge64_p3 P;
            ge64_from_p3(P, p);
            ge64_add_p3(acc[t], acc[t], P, d2);
        }
    }
    for (int d = threads / 2; d > 0; d /= 2)
        for (int t = 0; t < d; t++) ge64_add_p3(acc[t], acc[t], acc[t + d], d2);
    ge64_cmov_identity(acc[0], 1u - good);
    ge_p3 q;
    ge64_to_p3(q, acc[0]);
    encode(out, q, enc);
    return (int)good;
}

// the chunk plan of one level: start (nchunks + 1 values), base (m + 1), and nchunks, max_len, max_per_seg in info[0..2]
void h_plan(const uint64_t *offsets, size_t m, uint32_t chunk, uint32_t *start, uint32_t *base, uint32_t info[3])
{
    PsLevel L;
    ps_plan_level(L, offsets, m, chunk);
    memcpy(start, L.start.data(), L.start.size() * 4);
    memcpy(base, L.base.data(), L.base.size() * 4);
    info[0] = (uint32_t)L.start.size() - 1; info[1] = L.max_len; info[2] = L.max_per_seg;
}

// the pieces of whole chunks: returns the number of cuts written
size_t h_pieces(const uint32_t *start, size_t nchunks, uint32_t piece, uint32_t *cuts)
{
    std::vector<uint32_t> s(start, start + nchunks + 1), c;
    ps_pieces(c, s, piece);
    memcpy(cuts, c.data(), c.size() * 4);
    return c.size();
}
}
