/*
 * ed25519ph_oracle.c -- CPU restatement of ed25519-dalek's Ed25519ph (RFC 8032 5.1, phflag = 1) on the oracle library's
 * SHA-512, scalar and point code: SigningKey::sign_prehashed -> raw_sign_prehashed (E/signing.rs:312, :917-976) and
 * VerifyingKey::verify_prehashed / verify_prehashed_strict (E/verifying.rs:230-257, :424-459, RCompute :496-557).
 * TEST INFRASTRUCTURE ONLY: the parity source of the GPU Ed25519ph paths (tests/ed25519ph_oracle.py).  Compiled together
 * with the oracle sources, so the oracle library itself is unchanged.
 */
#include <string.h>

#include "oracle.h"

/* dom2(1, C) (E/signing.rs:945-951, E/verifying.rs:530-535) */
static void dom2(sha512_ctx *c, const uint8_t *ctx, size_t ctx_len)
{
    const uint8_t flag_len[2] = {1, (uint8_t)ctx_len};
    sha512_update(c, (const uint8_t *)"SigEd25519 no Ed25519 collisions", 32);
    sha512_update(c, flag_len, 2);
    sha512_update(c, ctx, ctx_len);
}

/* ExpandedSecretKey::from_bytes (E/hazmat.rs:84-99) */
static void expand(uint8_t a[32], uint8_t prefix[32], const uint8_t seed[32])
{
    uint8_t h[64];
    sha512(h, seed, 32);
    memcpy(a, h, 32); memcpy(prefix, h + 32, 32);
    a[0] &= 248; a[31] &= 127; a[31] |= 64;
}

/* raw_sign_prehashed; returns 5 (PrehashedContextLength) for a context longer than 255 bytes */
int ed25519ph_sign(uint8_t sig[64], const uint8_t prehash[64], const uint8_t *ctx, size_t ctx_len, const uint8_t seed[32])
{
    if (ctx_len > 255) return 5;
    uint8_t a[32], prefix[32], pk[32], h[64], r[32], k[32], ka[32], a_red[32];
    ge_p3 B, P;
    expand(a, prefix, seed);
    ge_basepoint(&B); ge_scalarmul(&P, a, &B); ge_compress(pk, &P);
    sha512_ctx c;
    sha512_init(&c); dom2(&c, ctx, ctx_len); sha512_update(&c, prefix, 32); sha512_update(&c, prehash, 64); sha512_final(&c, h);
    scalar_from_bytes_mod_order_wide(r, h);
    ge_scalarmul(&P, r, &B); ge_compress(sig, &P);
    sha512_init(&c); dom2(&c, ctx, ctx_len); sha512_update(&c, sig, 32); sha512_update(&c, pk, 32); sha512_update(&c, prehash, 64);
    sha512_final(&c, h);
    scalar_from_bytes_mod_order_wide(k, h);
    scalar_reduce(a_red, a);
    scalar_mul(ka, k, a_red);
    scalar_add(sig + 32, ka, r);
    return 0;
}

/* VerifyingKey::from_bytes, then verify_prehashed (strict = 0) or verify_prehashed_strict (strict = 1) */
int ed25519ph_verify(const uint8_t prehash[64], const uint8_t *ctx, size_t ctx_len, const uint8_t sig[64], const uint8_t pk[32],
                     int strict)
{
    ge_p3 A, R, minus_A, Rc;
    uint8_t h[64], k[32], expected[32];
    if (!ge_decompress(&A, pk)) return ED_ERR_POINT_DECOMPRESSION;
    if (!scalar_is_canonical(sig + 32)) return ED_ERR_SCALAR_FORMAT;
    if (strict) {
        if (!ge_decompress(&R, sig)) return ED_ERR_VERIFY;
        if (ge_is_small_order(&R) || ge_is_small_order(&A)) return ED_ERR_VERIFY;
    }
    sha512_ctx c;
    sha512_init(&c); dom2(&c, ctx, ctx_len); sha512_update(&c, sig, 32); sha512_update(&c, pk, 32); sha512_update(&c, prehash, 64);
    sha512_final(&c, h);
    scalar_from_bytes_mod_order_wide(k, h);
    ge_p3_neg(&minus_A, &A);
    edwards_vartime_double_scalar_mul_basepoint(&Rc, k, &minus_A, sig + 32);
    ge_compress(expected, &Rc);
    return memcmp(expected, sig, 32) == 0 ? ED_OK : ED_ERR_VERIFY;
}
