// Host build of the device code of the batched MSMs (msm_batch.cuh over fe64.cuh / ge64.cuh) with the operand-scale
// assertions of fe64.cuh and the limb-bound assertions of fe.cuh enabled, exported with a tiny C ABI for
// tests/test_msm_batch_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the chunk loops the kernels run keep every
// fe64_mul / fe64_sq operand within the scale rule and give the reference's bytes, and that the cut into chunks is the
// one the Python model describes.  Per-term preparation is what k_mb_prepare does (csrc/msm_batch.cu).
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/msm_batch.cuh"
#include <string.h>
#include <vector>

// 1 if T = XY / Z: the point handed to the next stage is a complete extended point (the next addition reads T)
static int t_consistent(const ge_p3 &q) { fe a, b; fe_mul(a, q.X, q.Y); fe_mul(b, q.Z, q.T); return fe_eq(a, b); }

extern "C" {
int h_mb_chunk_max(void) { return MB_CHUNK; }

// out = CompressedEdwardsY of sum s_t P_t over one chunk of len <= MB_CHUNK terms (32-byte scalars, CompressedEdwardsY
// points); ct: the constant-time loop.  Returns 1 if every point decodes (an undecodable one counts as the identity), 0 if
// not, -2 if the chunk's sum (which the per-MSM sum of the chunks adds) has T != XY / Z.
int h_mb_chunk(uint8_t *out, const uint8_t *scalars, const uint8_t *points, int len, int ct)
{
    std::vector<int8_t> digits((size_t)len * NAF_LEN + 4);
    std::vector<ge_pniels_packed> tables((size_t)len * 8 + 1);
    int all = 1;
    for (int t = 0; t < len; t++) {
        uint32_t s[8], e[8];
        memcpy(s, scalars + 32 * t, 32);
        memcpy(e, points + 32 * t, 32);
        ge_p3 p;
        const uint32_t good = ge_decompress_affine<1>(p.X, p.Y, e);
        fe_1(p.Z);
        fe_mul(p.T, p.X, p.Y);
        if (!good) { ge_p3_identity(p); all = 0; }
        ge64_p3 P;
        ge64_from_p3(P, p);
        if (ct) { mb_radix16(digits.data() + 64 * t, s); mb_table8(tables.data() + 8 * t, P); }
        else { naf5(digits.data() + NAF_LEN * t, s); straus_table5(tables.data() + 8 * t, P); }
    }
    ge64_p3 Q;
    if (ct) mb_chunk_ct(Q, digits.data(), tables.data(), (uint32_t)len);
    else mb_chunk_vt(Q, digits.data(), tables.data(), (uint32_t)len);
    ge_p3 q;
    ge64_to_p3(q, Q);
    uint32_t w[8];
    ge_compress<1>(w, q);
    memcpy(out, w, 32);
    return t_consistent(q) ? all : -2;
}

// The cut of nseg MSMs (nseg + 1 offsets) into chunks: chunk_base gets nseg + 1 slots; seg / first / len get one entry
// per chunk (capacity cap).  Returns the number of chunks.
uint32_t h_mb_tasks(const uint64_t *offsets, uint32_t nseg, uint32_t *chunk_base, uint32_t *seg, uint64_t *first, uint32_t *len,
                    uint32_t cap)
{
    uint32_t n = 0;
    for (uint32_t j = 0; j < nseg; j++) { chunk_base[j] = n; n += mb_chunks(offsets[j + 1] - offsets[j]); }
    chunk_base[nseg] = n;
    for (uint32_t c = 0; c < n && c < cap; c++) mb_task(seg[c], first[c], len[c], offsets, chunk_base, nseg, c);
    return n;
}

void h_mb_radix16(int8_t *d, const uint8_t *scalar)
{
    uint32_t s[8];
    memcpy(s, scalar, 32);
    mb_radix16(d, s);
}
}
