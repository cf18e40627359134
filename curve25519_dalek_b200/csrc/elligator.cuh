// elligator.cuh -- hashing into the group: the Ristretto Elligator map and RFC 9380 edwards25519_XMD:SHA-512_ELL2,
// one item per thread, host-compilable (the host build supplies the SHA-512 compression function).
//
//   ristretto_elligator       RistrettoPoint::elligator_ristretto_flavor      C/ristretto/elligator.rs:15-51
//   ristretto_from_uniform    RistrettoPoint::from_uniform_bytes              C/ristretto.rs:774-790
//   ristretto_hash_from_bytes RistrettoPoint::hash_from_bytes::<Sha512>       C/ristretto.rs:736-761
//   h2c_sha512_digest         its SHA-512 step, shared with Scalar::hash_from_bytes (scalars.cu)
//   ell2_encode               montgomery::elligator_encode (RFC 9380 G.2.1)   C/montgomery.rs:276-363
//   ell2_map_to_curve         EdwardsPoint::map_to_curve (rational map)       C/edwards.rs:651-686
//   h2c_from_bytes_wide       FieldElement::from_bytes_wide                   C/field.rs:110-147
//   xmd_sha512                expand_msg_xmd::<Sha512>, len_in_bytes 48, 96  C/field.rs:440-516
//   edwards_hash_to_curve<2>  EdwardsPoint::hash_to_curve::<Sha512>           C/edwards.rs:736-750
//   edwards_hash_to_curve<1>  EdwardsPoint::encode_to_curve::<Sha512>         C/edwards.rs:710-721
//
// Constant time, as the reference is with `subtle`: no branch, loop bound or address depends on message bytes or on a
// field value.  Message and DST lengths are public and set the block counts and where each byte of a hash input comes
// from.  The exceptional cases (Ns_D_is_sq, e1, e2, e3, tv1 == 0) are masked selects.  The exponentiations run on the
// FP64 field (fe_sqrt_ratio_i<1>, fe_pow_p58_f64, fe_invert_f64 through the compressions).
//
// Scale bookkeeping (fe.cuh:12-18): every input of a map is carried to scale 1; the comments give the scale of each
// sum or difference that feeds a multiplication.
#pragma once
#include "ge.cuh"

#if defined(__CUDACC__)
#include "hash.cuh"
#define H2C_FN __device__ __forceinline__
#else
#define H2C_FN inline
void h2c_host_sha512_compress(uint64_t h[8], uint64_t w[16]);   // supplied by the host build
#endif

H2C_FN void h2c_compress(uint64_t h[8], uint64_t w[16])
{
#if defined(__CUDACC__)
    sha512_compress_regs(h, w);
#else
    h2c_host_sha512_compress(h, w);
#endif
}

H2C_FN uint32_t h2c_bswap32(uint32_t x)
{
    return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
}

// SHA-512 of `total` input bytes, continuing from the chaining value h after `done` bytes.  With PRE the first 64
// input bytes are the eight big-endian words pre[]; every other byte q is byte_at(q).  The blocks are assembled in
// registers (static word indices); the block count and the source of each byte depend on the lengths only.
template <bool PRE, typename ByteAt>
H2C_FN void h2c_sha512(uint64_t h[8], size_t done, size_t total, const uint64_t *pre, ByteAt byte_at)
{
    const size_t nblocks = (total + 1 + 16 + 127) / 128;
#if defined(__CUDACC__)
#pragma unroll 1
#endif
    for (size_t blk = 0; blk < nblocks; blk++) {
        uint64_t w[16];
        const size_t base = blk * 128;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            uint64_t v = 0;
            if (PRE && blk == 0 && j < 8) {
                v = pre[j & 7];
            } else {
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    const size_t q = base + 8 * j + b;
                    const uint32_t byte = q < total ? (uint32_t)byte_at(q) : (q == total ? 0x80u : 0u);
                    v = (v << 8) | byte;
                }
            }
            w[j] = v;
        }
        if (blk == nblocks - 1) w[15] = (uint64_t)(done + total) * 8;   // w[14] stays 0: inputs < 2^61 bytes
        h2c_compress(h, w);
    }
}

H2C_FN void h2c_sha512_iv(uint64_t h[8])
{
    h[0] = 0x6a09e667f3bcc908ULL; h[1] = 0xbb67ae8584caa73bULL; h[2] = 0x3c6ef372fe94f82bULL; h[3] = 0xa54ff53a5f1d36f1ULL;
    h[4] = 0x510e527fade682d1ULL; h[5] = 0x9b05688c2b3e6c1fULL; h[6] = 0x1f83d9abfb41bd6bULL; h[7] = 0x5be0cd19137e2179ULL;
}

// 64 digest bytes (eight big-endian words) as 16 little-endian 32-bit words
H2C_FN void h2c_digest_words(uint32_t w[16], const uint64_t h[8])
{
#pragma unroll
    for (int i = 0; i < 8; i++) {
        w[2 * i] = h2c_bswap32((uint32_t)(h[i] >> 32));
        w[2 * i + 1] = h2c_bswap32((uint32_t)h[i]);
    }
}

// expand_msg_xmd::<Sha512> (C/field.rs:440-516, RFC 9380 5.3.1) for len_in_bytes = 48 COUNT (ell = COUNT):
// b1 = H(b0 || 1 || DST'), b2 = H((b0 ^ b1) || 2 || DST') with b0 = H(Z_pad || msg || I2OSP(48 COUNT, 2) || 0 || DST')
// and DST' = DST || I2OSP(dst_len, 1).  The Z_pad block is constant: b0 starts from SHA512_ZPAD_MIDSTATE.
template <int COUNT>
H2C_FN void xmd_sha512(uint64_t b1[8], uint64_t b2[8], const uint8_t *msg, size_t mlen, const uint8_t *dst, uint32_t dlen)
{
    const uint32_t lib = 48 * COUNT;
    auto dst_prime = [&](size_t k) -> uint32_t { return k < dlen ? dst[k] : dlen; };
    uint64_t b0[8];
#pragma unroll
    for (int i = 0; i < 8; i++) b0[i] = SHA512_ZPAD_MIDSTATE[i];
    h2c_sha512<false>(b0, 128, mlen + 4 + dlen, nullptr, [&](size_t q) -> uint32_t {
        if (q < mlen) return msg[q];
        const size_t r = q - mlen;
        return r == 0 ? lib >> 8 : (r == 1 ? lib & 0xffu : (r == 2 ? 0u : dst_prime(r - 3)));
    });
    h2c_sha512_iv(b1);
    h2c_sha512<true>(b1, 0, 64 + 1 + dlen + 1, b0, [&](size_t q) -> uint32_t { return q == 64 ? 1u : dst_prime(q - 65); });
    if (COUNT == 2) {
        uint64_t x[8];
#pragma unroll
        for (int i = 0; i < 8; i++) x[i] = b0[i] ^ b1[i];
        h2c_sha512_iv(b2);
        h2c_sha512<true>(b2, 0, 64 + 1 + dlen + 1, x, [&](size_t q) -> uint32_t { return q == 64 ? 2u : dst_prime(q - 65); });
    }
}

// FieldElement::from_bytes_wide (C/field.rs:110-147): 64 little-endian bytes (16 words) mod p.  The top bits of both
// halves are worth 2^255 = 19 and 2^511 = 722; the high half is worth 2^256 = 38.  Output scale 1.
H2C_FN void h2c_from_bytes_wide(fe &r, const uint32_t w[16])
{
    const uint32_t fl_top = w[7] >> 31, gl_top = w[15] >> 31;
    fe f, g;
    fe_frombytes_words(f, w);                        // bit 255 ignored
    fe_frombytes_words(g, w + 8);
    f.v[0] += 19u * fl_top + 722u * gl_top;
    fe_mul_small(g, g, 38);
    fe_add(r, f, g);
    fe_carry(r, r);
}

// hash_to_field's element i (C/field.rs:418-425): the 48 bytes uniform[48 i .. 48 i + 48) read big-endian, given as six
// big-endian words (w0 most significant), reversed into the low 48 bytes of from_bytes_wide's input.
H2C_FN void h2c_fe_from_be48(fe &r, uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3, uint64_t w4, uint64_t w5)
{
    const uint64_t L[6] = {w5, w4, w3, w2, w1, w0};
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 6; k++) { w[2 * k] = (uint32_t)L[k]; w[2 * k + 1] = (uint32_t)(L[k] >> 32); }
#pragma unroll
    for (int k = 12; k < 16; k++) w[k] = 0;
    h2c_from_bytes_wide(r, w);
}

// FieldElement::hash_to_field::<Sha512, COUNT> (C/field.rs:397-428)
template <int COUNT>
H2C_FN void h2c_hash_to_field(fe u[COUNT], const uint8_t *msg, size_t mlen, const uint8_t *dst, uint32_t dlen)
{
    uint64_t b1[8], b2[8];
    xmd_sha512<COUNT>(b1, b2, msg, mlen, dst, dlen);
    h2c_fe_from_be48(u[0], b1[0], b1[1], b1[2], b1[3], b1[4], b1[5]);
    if (COUNT == 2) h2c_fe_from_be48(u[COUNT - 1], b1[6], b1[7], b2[0], b2[1], b2[2], b2[3]);
}

// RistrettoPoint::elligator_ristretto_flavor (C/ristretto/elligator.rs:15-51); r0 scale 1.  D = 0 (r0 = +-sqrt(r / i)
// for r = -d or r = -1/d) reaches sqrt_ratio_i(N_s, 0), which gives (false, 0): the masked selects below take care of it.
H2C_FN void ristretto_elligator(ge_p3 &P, const fe &r0)
{
    fe i, d, one, c, r, t, t2, Ns, D, s, sp, Nt, ssq, k;
    fe_const_sqrtm1(i); fe_const_d(d); fe_1(one); fe_const_minus_one(c);
    fe_sq(t, r0); fe_mul(r, t, i);                   // r = i r0^2
    fe_add(t, r, one);                               // 2
    fe_const_one_minus_d_sq(k); fe_mul(Ns, t, k);    // N_s = (r + 1)(1 - d^2)
    fe_mul(t, d, r);
    fe_sub(t, c, t);                                 // 3   c - d r
    fe_add(t2, r, d);                                // 2   r + d
    fe_mul(D, t, t2);
    const uint32_t sq = fe_sqrt_ratio_i<1>(s, Ns, D);
    fe_mul(sp, s, r0);
    fe_cneg(sp, 1u - (uint32_t)fe_isnegative(sp));  // s' = -|s r0|
    fe_carry(sp, sp);
    fe_cmov(s, sp, 1u - sq);
    fe_cmov(c, r, 1u - sq);
    fe_sub(t, r, one);                               // 3
    fe_mul(t, c, t);
    fe_const_d_minus_one_sq(k); fe_mul(t, t, k);
    fe_sub(Nt, t, D);                                // 3   N_t = c (r - 1)(d - 1)^2 - D
    fe_sq(ssq, s);
    ge_p1p1 W;                                       // W_i is a completed point (elligator.rs:39-50)
    fe_add(t, s, s); fe_mul(W.X, t, D);              // X = 2 s D
    fe_const_sqrt_ad_minus_one(k); fe_mul(W.Z, Nt, k);   // Z = N_t sqrt(a d - 1)
    fe_sub(W.Y, one, ssq);                           // 3   Y = 1 - s^2
    fe_add(W.T, one, ssq);                           // 2   T = 1 + s^2
    ge_p1p1_to_p3(P, W);
}

// RistrettoPoint::from_uniform_bytes (C/ristretto.rs:774-790): 64 bytes as 16 little-endian words -> R_1 + R_2
H2C_FN void ristretto_from_uniform(ge_p3 &P, const uint32_t w[16])
{
    fe r1, r2;
    ge_p3 R1, R2;
    fe_frombytes_words(r1, w);                       // FieldElement::from_bytes: bit 255 ignored
    fe_frombytes_words(r2, w + 8);
    ristretto_elligator(R1, r1);
    ristretto_elligator(R2, r2);
    ge_add(P, R1, R2);
}

// SHA-512 of a message as 16 little-endian words: the 64 bytes that RistrettoPoint::hash_from_bytes (C/ristretto.rs:
// 736-761) and Scalar::hash_from_bytes (C/scalar.rs:617-624) feed to from_uniform_bytes and from_bytes_mod_order_wide
H2C_FN void h2c_sha512_digest(uint32_t w[16], const uint8_t *msg, size_t mlen)
{
    uint64_t h[8];
    h2c_sha512_iv(h);
    h2c_sha512<false>(h, 0, mlen, nullptr, [&](size_t q) -> uint32_t { return msg[q]; });
    h2c_digest_words(w, h);
}

// RistrettoPoint::hash_from_bytes::<Sha512> (C/ristretto.rs:736-761) -> CompressedRistretto as eight words
H2C_FN void ristretto_hash_from_bytes(uint32_t out[8], const uint8_t *msg, size_t mlen)
{
    uint32_t w[16];
    h2c_sha512_digest(w, msg, mlen);
    ge_p3 P;
    ristretto_from_uniform(P, w);
    ristretto_compress<1>(out, P);
}

// montgomery::elligator_encode (C/montgomery.rs:276-363, RFC 9380 G.2.1): (xn, xd, y) with the point (xn / xd, y) on
// curve25519 (yd = 1).  u scale 1; outputs scale 1.
H2C_FN void ell2_encode(fe &xn, fe &xd, fe &y, const fe &u)
{
    fe one, A, x1n, sm1, c2, tv1, tv2, tv3, gxd, gx1, gx2, y11, y12, y1, x2n, y21, y22, y2, ny;
    fe_1(one); fe_const_montgomery_a(A); fe_const_montgomery_a_neg(x1n); fe_const_sqrtm1(sm1); fe_const_ell2_c2(c2);
    fe_sq2(tv1, u); fe_carry(tv1, tv1);              // 1-2.  tv1 = 2 u^2
    fe_add(xd, one, tv1); fe_carry(xd, xd);          // 3.    xd = tv1 + 1
    fe_sq(tv2, xd);                                  // 5.
    fe_mul(gxd, tv2, xd);                            // 6.
    fe_mul(gx1, tv1, A);                             // 7.    gx1 = J tv1
    fe_mul(gx1, gx1, x1n);                           // 8.
    fe_add(gx1, gx1, tv2);                           // 9.    2
    fe_mul(gx1, gx1, x1n);                           // 10.
    fe_sq(tv3, gxd);                                 // 11.
    fe_sq(tv2, tv3);                                 // 12.
    fe_mul(tv3, tv3, gxd);                           // 13.
    fe_mul(tv3, tv3, gx1);                           // 14.
    fe_mul(tv2, tv2, tv3);                           // 15.
    fe_pow_p58_f64(y11, tv2);                        // 16.   y11 = tv2^c4
    fe_mul(y11, y11, tv3);                           // 17.
    fe_mul(y12, y11, sm1);                           // 18.
    fe_sq(tv2, y11); fe_mul(tv2, tv2, gxd);          // 19-20.
    const uint32_t e1 = (uint32_t)fe_eq(tv2, gx1);   // 21.
    y1 = y12; fe_cmov(y1, y11, e1);                  // 22.
    fe_mul(x2n, x1n, tv1);                           // 23.
    fe_mul(y21, y11, u);                             // 24.
    fe_mul(y21, y21, c2);                            // 25.
    fe_mul(y22, y21, sm1);                           // 26.
    fe_mul(gx2, gx1, tv1);                           // 27.
    fe_sq(tv2, y21); fe_mul(tv2, tv2, gxd);          // 28-29.
    const uint32_t e2 = (uint32_t)fe_eq(tv2, gx2);   // 30.
    y2 = y22; fe_cmov(y2, y21, e2);                  // 31.
    fe_sq(tv2, y1); fe_mul(tv2, tv2, gxd);           // 32-33.
    const uint32_t e3 = (uint32_t)fe_eq(tv2, gx1);   // 34.
    xn = x2n; fe_cmov(xn, x1n, e3);                  // 35.
    y = y2; fe_cmov(y, y1, e3);                      // 36.
    const uint32_t e4 = (uint32_t)fe_isnegative(y);  // 37.
    fe_neg(ny, y); fe_carry(ny, ny);
    fe_cmov(y, ny, e3 ^ e4);                         // 38.
}

// EdwardsPoint::map_to_curve (C/edwards.rs:651-686): elligator_encode, then the rational map of RFC 9380 D.1 to
// edwards25519 with its exceptional case tv1 = xd yd = 0 as a masked select.  yMd = 1, so xMn yMd is xMn.
H2C_FN void ell2_map_to_curve(ge_p3 &P, const fe &u)
{
    fe xMn, xMd, yMn, c1, xn, xd, yn, yd, tv1, zero, one;
    ell2_encode(xMn, xMd, yMn, u);
    fe_const_sqrtam2(c1); fe_0(zero); fe_1(one);
    fe_mul(xn, xMn, c1);                             // 2-3.  xn = xMn yMd c1
    fe_mul(xd, xMd, yMn);                            // 4.
    fe_sub(yn, xMn, xMd);                            // 5.    3
    fe_add(yd, xMn, xMd);                            // 6.    2
    fe_mul(tv1, xd, yd);                             // 7.
    const uint32_t e = (uint32_t)fe_iszero(tv1);     // 8.
    fe_cmov(xn, zero, e);                            // 9-12.
    fe_cmov(xd, one, e);
    fe_cmov(yn, one, e);
    fe_cmov(yd, one, e);
    fe_mul(P.X, xn, yd);
    fe_mul(P.Y, xd, yn);
    fe_mul(P.Z, xd, yd);
    fe_mul(P.T, xn, yn);
}

// EdwardsPoint::hash_to_curve::<Sha512> (COUNT = 2, C/edwards.rs:736-750) and encode_to_curve::<Sha512> (COUNT = 1,
// :710-721): maps, one addition for COUNT = 2, mul_by_cofactor (three doublings) -> CompressedEdwardsY words
template <int COUNT>
H2C_FN void edwards_hash_to_curve(uint32_t out[8], const uint8_t *msg, size_t mlen, const uint8_t *dst, uint32_t dlen)
{
    fe u[COUNT];
    h2c_hash_to_field<COUNT>(u, msg, mlen, dst, dlen);
    ge_p3 Q, R;
    ell2_map_to_curve(Q, u[0]);
    if (COUNT == 2) {
        ge_p3 Q1;
        ell2_map_to_curve(Q1, u[COUNT - 1]);
        ge_add(R, Q, Q1);
    } else {
        R = Q;
    }
    ge_mul_by_pow_2(Q, R, 3);                        // mul_by_cofactor (C/edwards.rs:1393-1395)
    ge_compress<1>(out, Q);
}
