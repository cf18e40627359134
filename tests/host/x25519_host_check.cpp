// Host build of the device X25519 ladder (x25519.cuh over fe64.cuh) with the operand-scale assertions of fe64.cuh and
// the limb-bound assertions of fe.cuh enabled, exported with a tiny C ABI for tests/test_x25519_host.py.
// TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the ladder the kernel runs keeps every
// fe64_mul / fe64_sq operand within the scale rule on every step and gives the reference's bytes.
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/x25519.cuh"
#include <string.h>

extern "C" {
// out = x25519(k, u); returns was_contributory
int h_x25519(uint8_t *out, const uint8_t *k, const uint8_t *u)
{
    uint32_t kw[8], uw[8], r[8];
    memcpy(kw, k, 32); memcpy(uw, u, 32);
    x25519_ladder(r, kw, uw);
    memcpy(out, r, 32);
    return (int)x25519_contributory(r);
}

// RFC 7748 5.2: k = u = 9, then `iterations` times (k, u) <- (x25519(k, u), k); out = the final k
void h_x25519_iterate(uint8_t *out, int iterations)
{
    uint32_t k[8] = {9, 0, 0, 0, 0, 0, 0, 0}, u[8] = {9, 0, 0, 0, 0, 0, 0, 0}, r[8];
    for (int it = 0; it < iterations; it++) {
        x25519_ladder(r, k, u);
        memcpy(u, k, 32);
        memcpy(k, r, 32);
    }
    memcpy(out, k, 32);
}
}
