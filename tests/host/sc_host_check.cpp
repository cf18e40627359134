// Host build of the device scalar arithmetic mod l (csrc/sc.cuh, built by a plain C++ compiler with SC_L / SC_MU as host
// constants), exported with a tiny C ABI for tests/test_sign_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product.
#include "../../curve25519_dalek_b200/csrc/sc.cuh"
#include <stddef.h>

extern "C" {
// n values each: x 16 words -> 8 words
void h_sc_reduce512(uint32_t *out, const uint32_t *x, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_reduce512(out + 8 * i, x + 16 * i);
}
void h_sc_mul(uint32_t *out, const uint32_t *a, const uint32_t *b, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_mul(out + 8 * i, a + 8 * i, b + 8 * i);
}
void h_sc_add(uint32_t *out, const uint32_t *a, const uint32_t *b, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_add(out + 8 * i, a + 8 * i, b + 8 * i);
}
void h_sc_neg(uint32_t *out, const uint32_t *a, size_t n)
{
    for (size_t i = 0; i < n; i++) sc_neg(out + 8 * i, a + 8 * i);
}
}
