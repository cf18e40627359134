// Host build of the scalar arithmetic of the batched Scalar calls (csrc/sc.cuh: sc_sub, sc_div_by_2, sc_is_canonical,
// sc_invert) and of the fold's chunk plan (csrc/ps_plan.h), exported with a tiny C ABI for tests/test_scalar_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product.
#include "../../curve25519_dalek_b200/csrc/ps_plan.h"
#include "../../curve25519_dalek_b200/csrc/sc.cuh"
#include <stddef.h>
#include <string.h>

extern "C" {
// n values each, 8 words in and out
void h_sc_sub(uint32_t *out, const uint32_t *a, const uint32_t *b, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_sub(out + 8 * i, a + 8 * i, b + 8 * i);
}
void h_sc_div_by_2(uint32_t *out, const uint32_t *a, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_div_by_2(out + 8 * i, a + 8 * i);
}
void h_sc_invert(uint32_t *out, const uint32_t *a, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_invert(out + 8 * i, a + 8 * i);
}
void h_sc_is_canonical(uint8_t *out, const uint32_t *a, size_t n)
{
    for (size_t i = 0; i < n; i++) out[i] = (uint8_t)sc_is_canonical(a + 8 * i);
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

int h_offsets_ok(const uint64_t *offsets, size_t m) { return ps_offsets_ok(offsets, m) ? 1 : 0; }
}
