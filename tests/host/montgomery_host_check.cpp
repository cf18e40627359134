// Host build of the device Montgomery ladder (mont_ladder<NW> of x25519.cuh over fe64.cuh) with the operand-scale
// assertions of fe64.cuh and the limb-bound assertions of fe.cuh enabled, exported with a tiny C ABI for
// tests/test_montgomery_host.py.  TEST INFRASTRUCTURE: not a CPU fallback of the product; it checks that the
// generalised ladder keeps every fe64_mul / fe64_sq operand within the scale rule for every bit length and gives the
// reference's bytes.
#define FE_CHECK_BOUNDS 1
#undef NDEBUG
#include "../../curve25519_dalek_b200/csrc/x25519.cuh"
#include <string.h>

extern "C" {
// out = u([b] P): b = bits nbits-1..0 of the int_bytes-byte little-endian integer `ints` (int_bytes <= 64), read into
// words as k_mont_ladder reads it (8 words up to 256 bits, else 16)
void h_mont_ladder(uint8_t *out, const uint8_t *ints, int int_bytes, int nbits, const uint8_t *u)
{
    uint32_t k[16] = {0}, uw[8], r[8];
    for (int j = 0; j < int_bytes; j++) k[j >> 2] |= (uint32_t)ints[j] << (8 * (j & 3));
    memcpy(uw, u, 32);
    if (nbits <= 256) mont_ladder<8>(r, k, nbits, uw);
    else mont_ladder<16>(r, k, nbits, uw);
    memcpy(out, r, 32);
}
}
