// codecs.cu -- batch wire-format codecs either side of the MSM (SURVEY 8f rank 2):
//   CompressedEdwardsY::decompress            C/edwards.rs:211-257        k_decompress_batch
//   EdwardsPoint::compress_batch              C/edwards.rs:619-647        k_compress_batch
//   CompressedRistretto::decompress           C/ristretto.rs:266-345      k_ristretto_decompress_batch
//   RistrettoPoint::double_and_compress_batch C/ristretto.rs:564-646      k_ristretto_double_and_compress_batch
//   EdwardsPoint::to_montgomery_batch         C/edwards.rs:592-612        k_to_montgomery_batch
// The two compressors and the Montgomery map use Montgomery's simultaneous inversion exactly like the reference
// (FieldElement::invert_batch, C/field.rs:239-274, zeros skipped): a thread owns CODEC_K consecutive points, so one
// 254-squaring inversion (on the FP64 field) is shared by CODEC_K points.
// Points travel as the reference's in-memory EdwardsPoint: 20 u64 limbs X | Y | Z | T in radix 2^51.
#include <algorithm>
#include <cstring>

#include "../../include/dalek_b200.h"
#include "engine.h"
#include "pieces.h"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

#define CODEC_K 8

__device__ __forceinline__ void load_limbs(fe &h, const uint64_t *__restrict__ src)
{
    uint64_t l[5];
#pragma unroll
    for (int k = 0; k < 5; k++) l[k] = src[k];
    fe_from_limbs51(h, l);
}
__device__ __forceinline__ void store_point(uint64_t *__restrict__ dst, const ge_p3 &p)
{
    uint64_t l[20];
    fe_to_limbs51(l, p.X); fe_to_limbs51(l + 5, p.Y); fe_to_limbs51(l + 10, p.Z); fe_to_limbs51(l + 15, p.T);
#pragma unroll
    for (int k = 0; k < 20; k++) dst[k] = l[k];
}

// in-place simultaneous inversion of v[0..CODEC_K), zeros stay zero (C/field.rs:239-274)
__device__ __forceinline__ void invert_batch(fe v[CODEC_K])
{
    fe scratch[CODEC_K], acc, t;
    fe_1(acc);
#pragma unroll
    for (int i = 0; i < CODEC_K; i++) {
        scratch[i] = acc;
        fe_mul(t, acc, v[i]);
        fe_cmov(acc, t, 1u - (uint32_t)fe_iszero(v[i]));
    }
    fe_invert_f64(acc, acc);
#pragma unroll
    for (int i = CODEC_K - 1; i >= 0; i--) {
        const uint32_t nz = 1u - (uint32_t)fe_iszero(v[i]);
        fe tmp, nv;
        fe_mul(tmp, acc, v[i]);
        fe_mul(nv, acc, scratch[i]);
        fe_cmov(v[i], nv, nz);
        fe_cmov(acc, tmp, nz);
    }
}

template <int F64>
__global__ void __launch_bounds__(128, 3)
k_decompress_batch(const uint32_t *__restrict__ in, size_t n, uint64_t *__restrict__ out, uint8_t *__restrict__ ok)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = in[8 * i + k];
    ge_p3 p;
    uint32_t good = ge_decompress_affine<F64>(p.X, p.Y, s);
    if (!good) { fe_0(p.X); fe_1(p.Y); }                  // None: the slot holds the identity
    fe_1(p.Z); fe_mul(p.T, p.X, p.Y);
    store_point(out + 20 * i, p);
    ok[i] = (uint8_t)good;
}

template <int F64>
__global__ void __launch_bounds__(128, 3)
k_ristretto_decompress_batch(const uint32_t *__restrict__ in, size_t n, uint64_t *__restrict__ out, uint8_t *__restrict__ ok)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = in[8 * i + k];
    ge_p3 p;
    uint32_t good = ristretto_decompress<F64>(p, s);
    if (!good) ge_p3_identity(p);
    store_point(out + 20 * i, p);
    ok[i] = (uint8_t)good;
}

// x = X/Z, y = Y/Z, bytes(y) with the sign of x in bit 255 (C/edwards.rs:619-631, affine.rs:71-75)
__global__ void __launch_bounds__(128)
k_compress_batch(const uint64_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i0 = t * CODEC_K;
    if (i0 >= n) return;
    fe z[CODEC_K];
#pragma unroll
    for (int k = 0; k < CODEC_K; k++) { if (i0 + k < n) load_limbs(z[k], in + 20 * (i0 + k) + 10); else fe_1(z[k]); }
    invert_batch(z);
#pragma unroll 1
    for (int k = 0; k < CODEC_K; k++) {
        if (i0 + k >= n) break;
        fe X, Y, x, y;
        load_limbs(X, in + 20 * (i0 + k)); load_limbs(Y, in + 20 * (i0 + k) + 5);
        fe_mul(x, X, z[k]); fe_mul(y, Y, z[k]);
        uint32_t w[8];
        fe_tobytes_words(w, y);
        w[7] ^= (uint32_t)fe_isnegative(x) << 31;
#pragma unroll
        for (int q = 0; q < 8; q++) out[8 * (i0 + k) + q] = w[q];
    }
}

// Montgomery u = (Z + Y) / (Z - Y) (C/edwards.rs:592-612), one shared inversion per CODEC_K points; the identity
// (Z = Y) has a zero denominator, skipped by invert_batch, and gives u = 0 like the reference's to_montgomery
__global__ void __launch_bounds__(128)
k_to_montgomery_batch(const uint64_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i0 = t * CODEC_K;
    if (i0 >= n) return;
    fe den[CODEC_K];
#pragma unroll
    for (int k = 0; k < CODEC_K; k++) {
        if (i0 + k < n) {
            fe Y, Z, d;
            load_limbs(Y, in + 20 * (i0 + k) + 5); load_limbs(Z, in + 20 * (i0 + k) + 10);
            fe_sub(d, Z, Y); fe_carry(den[k], d);
        } else fe_1(den[k]);
    }
    invert_batch(den);
#pragma unroll 1
    for (int k = 0; k < CODEC_K; k++) {
        if (i0 + k >= n) break;
        fe Y, Z, s, u;
        load_limbs(Y, in + 20 * (i0 + k) + 5); load_limbs(Z, in + 20 * (i0 + k) + 10);
        fe_add(s, Z, Y);
        fe_mul(u, s, den[k]);
        uint32_t w[8];
        fe_tobytes_words(w, u);
#pragma unroll
        for (int q = 0; q < 8; q++) out[8 * (i0 + k) + q] = w[q];
    }
}

// the per-point state of C/ristretto.rs:584-601
struct dbl_state { fe e, f, g, h, eg, fh; };
__device__ __forceinline__ void dbl_state_from(dbl_state &s, const uint64_t *__restrict__ pt)
{
    fe X, Y, Z, T, XX, YY, ZZ, dTT, d, t;
    load_limbs(X, pt); load_limbs(Y, pt + 5); load_limbs(Z, pt + 10); load_limbs(T, pt + 15);
    fe_const_d(d);
    fe_sq(XX, X); fe_sq(YY, Y); fe_sq(ZZ, Z);
    fe_sq(t, T); fe_mul(dTT, t, d);
    fe_add(t, Y, Y); fe_mul(s.e, X, t);                   // 2XY
    fe_add(t, ZZ, dTT); fe_carry(s.f, t);                 // Z^2 + dT^2
    fe_add(t, YY, XX); fe_carry(s.g, t);                  // Y^2 - aX^2
    fe_sub(t, ZZ, dTT); fe_carry(s.h, t);                 // Z^2 - dT^2
    fe_mul(s.eg, s.e, s.g);
    fe_mul(s.fh, s.f, s.h);
}

// compress(2 P) for every P, one shared inversion per CODEC_K points (C/ristretto.rs:604-645)
__global__ void __launch_bounds__(128)
k_ristretto_double_and_compress_batch(const uint64_t *__restrict__ in, size_t n, uint32_t *__restrict__ out)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, i0 = t * CODEC_K;
    if (i0 >= n) return;
    fe inv[CODEC_K];
#pragma unroll 1
    for (int k = 0; k < CODEC_K; k++) {
        if (i0 + k < n) { dbl_state s; dbl_state_from(s, in + 20 * (i0 + k)); fe_mul(inv[k], s.eg, s.fh); }
        else fe_1(inv[k]);
    }
    invert_batch(inv);
#pragma unroll 1
    for (int k = 0; k < CODEC_K; k++) {
        if (i0 + k >= n) break;
        dbl_state s;
        dbl_state_from(s, in + 20 * (i0 + k));            // recomputed: cheaper than keeping 6 elements x CODEC_K alive
        fe Zinv, Tinv, magic, sm1, t, minus_e, f_sqrta, e = s.e, g = s.g, h = s.h, enc;
        fe_const_invsqrt_a_minus_d(magic); fe_const_sqrtm1(sm1);
        fe_mul(Zinv, s.eg, inv[k]);
        fe_mul(Tinv, s.fh, inv[k]);
        fe_mul(t, s.eg, Zinv);
        const uint32_t negcheck1 = (uint32_t)fe_isnegative(t);
        fe_neg(minus_e, e); fe_carry(minus_e, minus_e);
        fe_mul(f_sqrta, s.f, sm1);
        fe_cmov(e, s.g, negcheck1);
        fe_cmov(g, minus_e, negcheck1);
        fe_cmov(h, f_sqrta, negcheck1);
        fe_cmov(magic, sm1, negcheck1);
        fe_mul(t, h, e); fe_mul(t, t, Zinv);
        const uint32_t negcheck2 = (uint32_t)fe_isnegative(t);
        fe_cneg(g, negcheck2); fe_carry(g, g);
        fe hg, gt;
        fe_sub(hg, h, g);                                  // scale 3
        fe_mul(gt, g, Tinv); fe_mul(gt, magic, gt);
        fe_mul(enc, hg, gt);
        fe_cneg(enc, (uint32_t)fe_isnegative(enc));
        uint32_t w[8];
        fe_tobytes_words(w, enc);
#pragma unroll
        for (int q = 0; q < 8; q++) out[8 * (i0 + k) + q] = w[q];
    }
}

void edwards_compress_enqueue(const uint64_t *d_limbs, size_t n, uint32_t *d_out, cudaStream_t st)
{
    k_compress_batch<<<cdiv(cdiv(n, CODEC_K), 128), 128, 0, st>>>(d_limbs, n, d_out);
}

extern "C" {

int dalek_b200_edwards_decompress_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint64_t *out_limbs, uint8_t *ok)
{
    if (!ctx || (n && (!in || !out_limbs || !ok))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    const bool f64 = ctx->opt_decompress_f64 != 0;
    int rc = run_pieces(ctx, nullptr, nullptr, in, 32, nullptr, 0, (uint8_t *)out_limbs, 160, ok, 1, n,
                        [&](const uint8_t *, const uint64_t *, const uint8_t *di, const uint8_t *, size_t m, uint8_t *d_o,
                            uint8_t *d_ok, cudaStream_t st) {
        if (f64) k_decompress_batch<1><<<cdiv(m, 128), 128, 0, st>>>((const uint32_t *)di, m, (uint64_t *)d_o, d_ok);
        else k_decompress_batch<0><<<cdiv(m, 128), 128, 0, st>>>((const uint32_t *)di, m, (uint64_t *)d_o, d_ok);
        return 0;
    });
    if (rc) return rc;
    uint8_t all = 1;
    for (size_t i = 0; i < n; i++) all &= ok[i];
    return all ? DALEK_OK : DALEK_NONE;
}

int dalek_b200_ristretto_decompress_batch(dalek_b200_ctx *ctx, const uint8_t *in, size_t n, uint64_t *out_limbs, uint8_t *ok)
{
    if (!ctx || (n && (!in || !out_limbs || !ok))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    const bool f64 = ctx->opt_decompress_f64 != 0;
    int rc = run_pieces(ctx, nullptr, nullptr, in, 32, nullptr, 0, (uint8_t *)out_limbs, 160, ok, 1, n,
                        [&](const uint8_t *, const uint64_t *, const uint8_t *di, const uint8_t *, size_t m, uint8_t *d_o,
                            uint8_t *d_ok, cudaStream_t st) {
        if (f64) k_ristretto_decompress_batch<1><<<cdiv(m, 128), 128, 0, st>>>((const uint32_t *)di, m, (uint64_t *)d_o, d_ok);
        else k_ristretto_decompress_batch<0><<<cdiv(m, 128), 128, 0, st>>>((const uint32_t *)di, m, (uint64_t *)d_o, d_ok);
        return 0;
    });
    if (rc) return rc;
    uint8_t all = 1;
    for (size_t i = 0; i < n; i++) all &= ok[i];
    return all ? DALEK_OK : DALEK_NONE;
}

int dalek_b200_edwards_compress_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!limbs || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    return run_pieces(ctx, nullptr, nullptr, (const uint8_t *)limbs, 160, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *, const uint64_t *, const uint8_t *di, const uint8_t *, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st) {
        k_compress_batch<<<cdiv(cdiv(m, CODEC_K), 128), 128, 0, st>>>((const uint64_t *)di, m, (uint32_t *)d_o);
        return 0;
    });
}

int dalek_b200_ristretto_double_and_compress_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!limbs || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    return run_pieces(ctx, nullptr, nullptr, (const uint8_t *)limbs, 160, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *, const uint64_t *, const uint8_t *di, const uint8_t *, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st) {
        k_ristretto_double_and_compress_batch<<<cdiv(cdiv(m, CODEC_K), 128), 128, 0, st>>>((const uint64_t *)di, m, (uint32_t *)d_o);
        return 0;
    });
}

int dalek_b200_edwards_to_montgomery_batch(dalek_b200_ctx *ctx, const uint64_t *limbs, size_t n, uint8_t *out)
{
    if (!ctx || (n && (!limbs || !out))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return run_pieces(ctx, nullptr, nullptr, (const uint8_t *)limbs, 160, nullptr, 0, out, 32, nullptr, 0, n,
                      [&](const uint8_t *, const uint64_t *, const uint8_t *di, const uint8_t *, size_t m, uint8_t *d_o,
                          uint8_t *, cudaStream_t st) {
        k_to_montgomery_batch<<<cdiv(cdiv(m, CODEC_K), 128), 128, 0, st>>>((const uint64_t *)di, m, (uint32_t *)d_o);
        return 0;
    });
}

}  // extern "C"
