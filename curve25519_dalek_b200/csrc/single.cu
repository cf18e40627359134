// single.cu -- many independent Ed25519 verifications, one verdict per signature (SURVEY 8f rank 3):
//   VerifyingKey::from_bytes + verify        ed25519-dalek/src/verifying.rs:167-175, :203-219
//   VerifyingKey::verify_strict              ed25519-dalek/src/verifying.rs:359-382
//   RCompute                                 ed25519-dalek/src/verifying.rs:496-557
//   verify_prehashed[_strict]                ed25519-dalek/src/verifying.rs:230-257, :424-459 (the same paths with the
//                                            Ed25519ph challenge SHA-512(dom2 || R || A || PH): k_verify_each_ph, k_hram_ph)
//   EdwardsPoint::vartime_double_scalar_mul_basepoint   curve25519-dalek/src/edwards.rs:1388-1397
//       (serial backend scalar_mul/vartime_double_base.rs:23-72)
// Unlike verify_batch, `verify` recomputes R' = [s]B - [k]A and compares its ENCODING with the signature's R
// bytes, so a non-canonical R fails here although it passes the batch equation (ed25519-dalek README,
// "Validation criteria"); VALIDATIONVECTORS pins both behaviours (tests).
//
// Two paths, same results.  When the keys of a call repeat, the doublings are paid once per KEY (per-key comb tables,
// k_each_key_* and k_verify_each_comb below: 128 mixed additions per signature, no doubling).  Otherwise (plain kernel,
// k_verify_each): one thread per signature.  [s]B + [k](-A) is computed on the FP64 field by double_base_eval
// (double_base.cuh, shared with the double-base batch of double_base.cu): radix-16 signed digits (scalar.rs:1019-1051),
// 63 x 4 doublings, 64 mixed additions from the shared 8-entry table of B and 64 additions from the thread's own 8-entry
// table of -A (local memory).  The reference interleaves width-5 / width-8 NAFs; fixed radix-16 keeps the lanes of a
// warp on the same schedule.  Same group element, hence the same encoding.
#include <algorithm>
#include <cstring>
#include <new>

#include "../../include/dalek_b200.h"
#include "double_base.cuh"
#include "engine.h"
#include "ge64.cuh"
#include "hash.cuh"
#include "pieces.h"
#include "sc.cuh"

static inline unsigned cdiv(size_t a, unsigned b) { return (unsigned)((a + b - 1) / b); }

// [8]P == identity  (EdwardsPoint::is_small_order, C/edwards.rs:1405-1407)
__device__ __forceinline__ uint32_t is_small_order(const ge_p3 &p)
{
    ge_p3 q;
    ge_mul_by_pow_2(q, p, 3);
    return ge_is_identity(q);
}

#ifndef EACH_MIN_BLOCKS
#define EACH_MIN_BLOCKS 2
#endif
// PH = 0: k = SHA-512(R || A || M), message i at msgs + offs[i]; PH = 1 (Ed25519ph, verifying.rs:530-535): k =
// SHA-512(dom2 || R || A || PH), prehash i at msgs + 64 i (offs unused).  Everything after the challenge is shared.
template <int PH>
__device__ __forceinline__ void verify_each_body(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs,
                                                 const Sha512Prefix *dom, const uint32_t *__restrict__ sigs,
                                                 const uint32_t *__restrict__ keys, size_t n, int strict,
                                                 const ge_niels_packed *__restrict__ base_row0, uint8_t *__restrict__ out)
{
    __shared__ double s_B[8 * 15];                               // (j+1) B as balanced FP64 affine Niels, j = 0..7
    if (threadIdx.x < 8) double_base_stage_B(s_B + 15 * threadIdx.x, base_row0[threadIdx.x]);
    __syncthreads();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t R[8], s[8], Ak[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { R[k] = sigs[16 * i + k]; s[k] = sigs[16 * i + 8 + k]; Ak[k] = keys[8 * i + k]; }
    // k = SHA-512(R || A || M) mod l  (verifying.rs:515-523)
    uint32_t h[8];
    {
        uint32_t dig[16];
        if (PH) sha512_pxm<2, 1>(dig, dom->b, dom->len, R, Ak, msgs + 64 * i, 64);
        else {
            const uint64_t lo = offs[i], hi = offs[i + 1];
            sha512_ram(dig, R, Ak, msgs + lo, (size_t)(hi - lo));
        }
        sc_reduce512(h, dig);
    }
    ge_p3 A;
    fe_1(A.Z);
    const uint32_t okA = ge_decompress_affine<1>(A.X, A.Y, Ak);               // verifying.rs:167-175
    if (!okA) { fe_0(A.X); fe_1(A.Y); }
    fe_mul(A.T, A.X, A.Y);
    const uint32_t okS = sc_is_canonical(s);                                  // signature.rs:89-94, :149-169
    uint32_t okR = 1, small = 0;
    if (strict) {                                                             // verifying.rs:366-376
        ge_p3 Rp;
        fe_1(Rp.Z);
        okR = ge_decompress_affine<1>(Rp.X, Rp.Y, R);
        if (!okR) { fe_0(Rp.X); fe_1(Rp.Y); }
        fe_mul(Rp.T, Rp.X, Rp.Y);
        small = is_small_order(Rp) | is_small_order(A);
    }
    if (!okS) {                                                               // keep the digits in range; the verdict is fixed below
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = 0;
    }
    // [k](-A) + [s]B
    ge_p3 nA = A;
    fe_neg(nA.X, A.X); fe_carry(nA.X, nA.X);
    fe_neg(nA.T, A.T); fe_carry(nA.T, nA.T);
    ge64_p3 acc;
    DoubleBaseLocal w;
    double_base_eval(acc, nA, h, s, s_B, w);
    ge_p3 Rc; ge64_to_p3(Rc, acc);
    uint32_t enc[8];
    ge_compress<1>(enc, Rc);                                                  // RCompute::finish, verifying.rs:553-556
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) diff |= enc[k] ^ R[k];
    // precedence: key decoding happens in from_bytes, before verify can be called; then the s check of
    // Signature parsing; then everything else is a Verify error
    uint8_t v = ED25519_ERR_VERIFY;
    if (!okA) v = ED25519_ERR_POINT_DECOMPRESSION;
    else if (!okS) v = ED25519_ERR_SCALAR_FORMAT;
    else if (okR && !small && diff == 0) v = DALEK_OK;
    out[i] = v;
}

__global__ void __launch_bounds__(128, EACH_MIN_BLOCKS)
k_verify_each(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ sigs,
              const uint32_t *__restrict__ keys, size_t n, int strict, const ge_niels_packed *__restrict__ base_row0,
              uint8_t *__restrict__ out)
{
    verify_each_body<0>(msgs, offs, nullptr, sigs, keys, n, strict, base_row0, out);
}

// Ed25519ph: phs holds n 64-byte prehashes
__global__ void __launch_bounds__(128, EACH_MIN_BLOCKS)
k_verify_each_ph(const uint8_t *__restrict__ phs, const __grid_constant__ Sha512Prefix dom, const uint32_t *__restrict__ sigs,
                 const uint32_t *__restrict__ keys, size_t n, int strict, const ge_niels_packed *__restrict__ base_row0,
                 uint8_t *__restrict__ out)
{
    verify_each_body<1>(phs, nullptr, &dom, sigs, keys, n, strict, base_row0, out);
}

static int verify_each_dev(dalek_b200_ctx *ctx, const uint8_t *d_msgs, const uint64_t *d_offs, const uint32_t *d_sigs,
                           const uint32_t *d_keys, size_t n, int strict, uint8_t *d_out, const Sha512Prefix *ph_dom)
{
    if (!n) return 0;
    cudaStream_t st = ctx->stream;
    const ge_niels_packed *base = (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p;
    if (ph_dom) k_verify_each_ph<<<cdiv(n, 128), 128, 0, st>>>(d_msgs, *ph_dom, d_sigs, d_keys, n, strict, base, d_out);
    else k_verify_each<<<cdiv(n, 128), 128, 0, st>>>(d_msgs, d_offs, d_sigs, d_keys, n, strict, base, d_out);
    ctx->launches++;
    CUDA_TRY(ctx, cudaGetLastError());
    return 0;
}

// ---- keys that sign many signatures: per-key comb tables ----------------------------------------------------------
// R' = [s]B - [k]A costs 252 doublings because A is only known when the call arrives.  When the batch holds few distinct
// keys (a validator set, an exchange's hot keys: bench.py's 2^22 signatures come from 1024 keys), the doublings can be
// paid once per KEY: with the 64 x 8 multiples (j+1) 16^i A of every distinct key in device memory (the fixed-base table
// of B has the same shape), [s]B - [k]A = sum_i s_i (16^i B) - k_i (16^i A) over radix-16 signed digits is 128 mixed
// additions and no doubling -- the comb of k_double_base_comb (straus.cu) with one table gathered per signature.  Same
// group element as the reference's vartime_double_scalar_mul_basepoint, hence the same encoding and verdict; keys are
// de-duplicated, decompressed and tabulated once per call (16 KiB x 4 = 64 KiB of table per key: 1024 keys
// make 64 MB, more than the 50 MB L2 of an H100, so part of the gathers reach HBM; measured on an H100, that costs
// a few percent against L2-resident tables, far less than the plain kernel loses: profiles/each_keys_h100.json).
#define EACH_K 4                        // signatures per thread of the comb kernel: one shared inversion
#define EACH_ENT 16                     // doubles per table entry: y+x | y-x | 2dxy as balanced limbs, padded to 128 bytes
#define EACH_KEY_DOUBLES (64 * 8 * EACH_ENT)
#define EACH_COMB_SMEM (COMB_BASE_DOUBLES * sizeof(double))   // k_verify_each_comb: the 64 x 8 x 15 table of B (60 KiB)

// one thread per distinct key: decompress, 16^i A for i = 0..63 (63 x 4 doublings), small-order mark
__global__ void __launch_bounds__(64)
k_each_key_pow16(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ uniq, size_t nkeys, ge_p3_raw *__restrict__ pw,
                 uint8_t *__restrict__ kstat)
{
    const size_t slot = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= nkeys) return;
    const size_t i = uniq[slot];
    uint32_t Ak[8];
#pragma unroll
    for (int k = 0; k < 8; k++) Ak[k] = keys[8 * i + k];
    ge_p3 A;
    fe_1(A.Z);
    const uint32_t ok = ge_decompress_affine<1>(A.X, A.Y, Ak);             // verifying.rs:167-175
    if (!ok) { fe_0(A.X); fe_1(A.Y); }
    fe_mul(A.T, A.X, A.Y);
    kstat[slot] = (uint8_t)((ok ? 0 : 1) | (is_small_order(A) ? 2 : 0));
    ge64_p3 P; ge64_from_p3(P, A);
#pragma unroll 1
    for (int pos = 0; pos < 64; pos++) {
        if (pos) { ge64_dbl(P, P); ge64_dbl(P, P); ge64_dbl(P, P); ge64_dbl(P, P); }
        ge_p3 q; ge64_to_p3(q, P);
        ge_p3_raw r; ge_p3_store_raw(r, q);
        uint4 *o = reinterpret_cast<uint4 *>(pw + slot * 64 + pos);
#pragma unroll
        for (int w = 0; w < 10; w++) o[w] = make_uint4(r.w[4 * w], r.w[4 * w + 1], r.w[4 * w + 2], r.w[4 * w + 3]);
    }
}

// one thread per table entry: (j+1) 16^i A as affine Niels coordinates in balanced FP64 limbs
__global__ void __launch_bounds__(128)
k_each_key_rows(const ge_p3_raw *__restrict__ pw, size_t nkeys, double *__restrict__ tab)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nkeys * 512) return;
    const int j = (int)(t & 7);
    ge_p3 P;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(pw + (t >> 3));
        ge_p3_raw r;
#pragma unroll
        for (int w = 0; w < 10; w++) { uint4 v = src[w]; r.w[4 * w] = v.x; r.w[4 * w + 1] = v.y; r.w[4 * w + 2] = v.z; r.w[4 * w + 3] = v.w; }
        ge_p3_load_raw(P, r);
    }
    ge_pniels nb; ge_p3_to_pniels(nb, P);
    ge_p3 Q = P;
#pragma unroll 1
    for (int k = 0; k < j; k++) ge_padd(Q, Q, nb, 0);                      // (j+1) * 16^i A
    fe zi, x, y;
    fe_invert_f64(zi, Q.Z);
    fe_mul(x, Q.X, zi); fe_mul(y, Q.Y, zi);
    ge_niels nl; ge_affine_to_niels(nl, x, y);
    fe64 e[3];
    fe64_from_fe(e[0], nl.ypx); fe64_from_fe(e[1], nl.ymx); fe64_from_fe(e[2], nl.xy2d);
    double *dst = tab + t * EACH_ENT;
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int k = 0; k < 5; k++) dst[5 * c + k] = e[c].v[k];
    dst[15] = 0.0;
}

// The y coordinates of the eight points of small order (identity, order 2, order 4 twice, order 8 four times), canonical:
// 1, -1, 0, y8, -y8 (constants::EIGHT_TORSION, u64/constants.rs:196-340).  verify_strict rejects a signature whose R is one of
// them (verifying.rs:366-376); once the encodings of R' and R agree, R's bytes are canonical and a comparison of bytes decides.
__constant__ uint32_t c_small_y[5][8] = {
    {0x00000001u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
    {0xffffffecu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x7fffffffu},
    {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
    {0x706a17c7u, 0x4fd84d3du, 0x760b3cbau, 0x0f67100du, 0xfa53202au, 0xc6cc392cu, 0x77fdc74eu, 0x7a03ac92u},
    {0x8f95e826u, 0xb027b2c2u, 0x89f4c345u, 0xf098eff2u, 0x05acdfd5u, 0x3933c6d3u, 0x880238b1u, 0x05fc536du}};

// one thread per signature: 64 additions from B's table (shared memory) and 64 from the key's table (L2), compress, compare
__global__ void __launch_bounds__(128, 3)
k_verify_each_comb(const uint32_t *__restrict__ sigs, const uint32_t *__restrict__ hs, const uint8_t *__restrict__ bad_s,
                   const uint32_t *__restrict__ rep, const uint32_t *__restrict__ dense, const uint8_t *__restrict__ kstat,
                   const double *__restrict__ tab, const ge_niels_packed *__restrict__ base_table, size_t i0, size_t n, int strict,
                   uint8_t *__restrict__ out)
{
    extern __shared__ double s_B[];                                        // 64 x 8 x 15: (j+1) 16^i B as balanced limbs
    for (int e = threadIdx.x; e < 512; e += blockDim.x) {
        ge64_niels q; ge64_niels_unpack(q, base_table[e]);
        fe64 c;
        double *dst = s_B + 15 * e;
        fe64_carry(c, q.ypx);  for (int k = 0; k < 5; k++) dst[k] = c.v[k];
        fe64_carry(c, q.ymx);  for (int k = 0; k < 5; k++) dst[5 + k] = c.v[k];
        fe64_carry(c, q.xy2d); for (int k = 0; k < 5; k++) dst[10 + k] = c.v[k];
    }
    __syncthreads();
    // EACH_K consecutive signatures per thread: their EACH_K inversions (the x / Z, y / Z of the encodings) become one, by
    // the simultaneous-inversion pattern of field.rs:239-273 -- 265 field operations per signature become 265 / 4 + 3
    const size_t first = i0 + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * EACH_K;
    if (first >= n) return;
    fe PX[EACH_K], PY[EACH_K], PZ[EACH_K], pre[EACH_K];
    uint8_t pending[EACH_K];
#pragma unroll 1
    for (int q = 0; q < EACH_K; q++) {
        const size_t i = first + q;
        if (i >= n) { fe_0(PX[q]); fe_1(PY[q]); fe_1(PZ[q]); pending[q] = 0xff; continue; }
        uint32_t s[8], h[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { s[k] = sigs[16 * i + 8 + k]; h[k] = hs[8 * i + k]; }
        const uint32_t okS = !bad_s[i];
        if (!okS) {                                                        // keep the digits in range; the verdict is fixed below
#pragma unroll
            for (int k = 0; k < 8; k++) s[k] = 0;
        }
        const uint32_t slot = dense[rep[i]];
        const uint32_t ks = kstat[slot];
        const double2 *TA = reinterpret_cast<const double2 *>(tab + (size_t)slot * EACH_KEY_DOUBLES);
        ge64_p3 acc; ge64_identity(acc);
        int cs = 0, ch = 0;                                                // radix-16 recoding carries (scalar.rs:1040-1046)
        uint32_t ws = 0, wh = 0;
#pragma unroll 1
        for (int pos = 0; pos < 64; pos++) {
            if ((pos & 7) == 0) { ws = s[pos >> 3]; wh = h[pos >> 3]; }
            int dsg = (int)(ws & 15) + cs; ws >>= 4;
            int dhg = (int)(wh & 15) + ch; wh >>= 4;
            if (pos < 63) { cs = (dsg + 8) >> 4; dsg -= cs << 4; ch = (dhg + 8) >> 4; dhg -= ch << 4; }
            // the key's entry first: its L2 latency runs under the addition from B's table
            double2 a2[8];
            const int mh = dhg < 0 ? -dhg : dhg;
            if (mh) {
                const double2 *src = TA + ((size_t)pos * 8 + (mh - 1)) * (EACH_ENT / 2);
#pragma unroll
                for (int k = 0; k < 8; k++) a2[k] = __ldg(src + k);
            }
            if (dsg) {
                const int m = dsg < 0 ? -dsg : dsg;
                const double *row = s_B + 15 * (8 * pos + (m - 1));
                ge64_niels qn;
#pragma unroll
                for (int k = 0; k < 5; k++) { qn.ypx.v[k] = row[k]; qn.ymx.v[k] = row[5 + k]; qn.xy2d.v[k] = row[10 + k]; }
                ge64_madd(acc, acc, qn, (uint32_t)(dsg < 0));
            }
            if (mh) {
                ge64_niels qn;
                qn.ypx.v[0] = a2[0].x; qn.ypx.v[1] = a2[0].y; qn.ypx.v[2] = a2[1].x; qn.ypx.v[3] = a2[1].y; qn.ypx.v[4] = a2[2].x;
                qn.ymx.v[0] = a2[2].y; qn.ymx.v[1] = a2[3].x; qn.ymx.v[2] = a2[3].y; qn.ymx.v[3] = a2[4].x; qn.ymx.v[4] = a2[4].y;
                qn.xy2d.v[0] = a2[5].x; qn.xy2d.v[1] = a2[5].y; qn.xy2d.v[2] = a2[6].x; qn.xy2d.v[3] = a2[6].y; qn.xy2d.v[4] = a2[7].x;
                ge64_madd(acc, acc, qn, (uint32_t)(dhg > 0));               // minus [k] A: positive digits subtract
            }
        }
        ge_p3 Rc; ge64_to_p3(Rc, acc);
        PX[q] = Rc.X; PY[q] = Rc.Y; PZ[q] = Rc.Z;
        pending[q] = (uint8_t)((ks & 1) ? ED25519_ERR_POINT_DECOMPRESSION : !okS ? ED25519_ERR_SCALAR_FORMAT : ((strict && (ks & 2)) ? ED25519_ERR_VERIFY : 0));
    }
    // 1 / Z of the EACH_K points with one inversion (Z is never zero: the formulas are complete)
    fe run; fe_copy(run, PZ[0]);
#pragma unroll 1
    for (int q = 1; q < EACH_K; q++) { fe_copy(pre[q], run); fe_mul(run, run, PZ[q]); }
    fe inv; fe_invert_f64(inv, run);
#pragma unroll 1
    for (int q = EACH_K - 1; q >= 0; q--) {
        fe zi;
        if (q) { fe_mul(zi, inv, pre[q]); fe_mul(inv, inv, PZ[q]); } else fe_copy(zi, inv);
        const size_t i = first + q;
        if (i >= n) continue;
        fe x, y;
        fe_mul(x, PX[q], zi); fe_mul(y, PY[q], zi);
        uint32_t enc[8];
        fe_tobytes_words(enc, y);                                          // RCompute::finish, verifying.rs:553-556 (EdwardsPoint::compress)
        enc[7] ^= (uint32_t)fe_isnegative(x) << 31;
        uint32_t R[8], diff = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { R[k] = sigs[16 * i + k]; diff |= enc[k] ^ R[k]; }
        uint32_t small = 0;
        if (strict) {                                                      // verifying.rs:366-376: R of small order (A: per key, above)
#pragma unroll 1
            for (int t = 0; t < 5; t++) {
                uint32_t d = (R[7] & 0x7fffffffu) ^ c_small_y[t][7];
#pragma unroll
                for (int k = 0; k < 7; k++) d |= R[k] ^ c_small_y[t][k];
                small |= (uint32_t)(d == 0);
            }
        }
        out[i] = pending[q] ? pending[q] : (uint8_t)((diff == 0 && !small) ? DALEK_OK : ED25519_ERR_VERIFY);
    }
}

// Verification (verify or verify_strict) of n signatures (device inputs) through per-key comb tables; *used = 0 if the keys do not repeat
// enough (or the tables would not fit) and the caller should run k_verify_each instead.  ph_dom: Ed25519ph (d_msgs = n prehashes).
static int verify_each_comb(dalek_b200_ctx *ctx, const uint8_t *d_msgs, const uint64_t *d_offs, const uint32_t *d_sigs,
                            const uint32_t *d_keys, size_t n, int strict, uint8_t *d_out, bool *used, const Sha512Prefix *ph_dom)
{
    *used = false;
    if (!n || !ctx->opt_each_comb || !ctx->opt_field_f64) return 0;
    int rc;
    EachFront f;
    if ((rc = verify_each_front(ctx, d_msgs, d_offs, d_sigs, d_keys, n, &f, ph_dom))) return rc;
    const size_t tab_bytes = f.nkeys * EACH_KEY_DOUBLES * sizeof(double);
    if (tab_bytes > ((size_t)8 << 30)) return 0;
    if (ctx->opt_each_comb == 1 && f.nkeys * 8 > n) return 0;             // a table costs about what eight plain verifications cost
    cudaStream_t st = ctx->stream;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_EACH_POW], f.nkeys * 64 * sizeof(ge_p3_raw)))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_EACH_TABLES], tab_bytes))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_EACH_KEY_STATUS], f.nkeys))) return rc;
    k_each_key_pow16<<<cdiv(f.nkeys, 64), 64, 0, st>>>(d_keys, f.uniq, f.nkeys, (ge_p3_raw *)ctx->ws[WS_EACH_POW].p, (uint8_t *)ctx->ws[WS_EACH_KEY_STATUS].p);
    k_each_key_rows<<<cdiv(f.nkeys * 512, 128), 128, 0, st>>>((const ge_p3_raw *)ctx->ws[WS_EACH_POW].p, f.nkeys, (double *)ctx->ws[WS_EACH_TABLES].p);
    if (!ctx->each_attr_set) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(k_verify_each_comb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EACH_COMB_SMEM));
        ctx->each_attr_set = true;
    }
    k_verify_each_comb<<<cdiv((n + EACH_K - 1) / EACH_K, 128), 128, EACH_COMB_SMEM, st>>>(d_sigs, f.hs, f.bad_s, f.rep, f.dense, (const uint8_t *)ctx->ws[WS_EACH_KEY_STATUS].p,
                                                       (const double *)ctx->ws[WS_EACH_TABLES].p, (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p, 0, n, strict, d_out);
    ctx->launches += 3;
    CUDA_TRY(ctx, cudaGetLastError());
    *used = true;
    return 0;
}

// the return code of a per-signature call: Verify if any signature failed
static int verify_each_summary(const uint8_t *results, size_t n)
{
    uint8_t any = 0;
    for (size_t i = 0; i < n; i++) any |= results[i];
    return any ? ED25519_ERR_VERIFY : DALEK_OK;
}

// The rest of a per-signature call whose inputs are in device memory: the per-key comb path, or the plain kernel when
// the keys do not repeat enough; then the results are read back.  ph_dom: Ed25519ph (d_msgs = n prehashes).
static int verify_each_resident(dalek_b200_ctx *ctx, const uint8_t *d_msgs, const uint64_t *d_offs, const uint32_t *d_sigs,
                                const uint32_t *d_keys, size_t n, int strict, const Sha512Prefix *ph_dom, uint8_t *results)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_ITEM_STATUS], std::max<size_t>(1, n)))) return rc;
    uint8_t *d_out = (uint8_t *)ctx->ws[WS_ITEM_STATUS].p;
    bool comb = false;
    if ((rc = verify_each_comb(ctx, d_msgs, d_offs, d_sigs, d_keys, n, strict, d_out, &comb, ph_dom))) return rc;
    if (!comb && (rc = verify_each_dev(ctx, d_msgs, d_offs, d_sigs, d_keys, n, strict, d_out, ph_dom))) return rc;
    if (n) CUDA_TRY(ctx, cudaMemcpyAsync(results, d_out, n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return verify_each_summary(results, n);
}

extern "C" {

int ed25519_b200_verify_each_flat_dev(dalek_b200_ctx *ctx, const void *d_msgs_flat, const void *d_msg_offsets, const void *d_sigs,
                                      const void *d_pubkeys, size_t n, int strict, uint8_t *results)
{
    if (!ctx || (n && (!d_msg_offsets || !d_sigs || !d_pubkeys || !results))) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    if ((rc = base_table_ensure(ctx))) return rc;
    return verify_each_resident(ctx, (const uint8_t *)d_msgs_flat, (const uint64_t *)d_msg_offsets, (const uint32_t *)d_sigs,
                                (const uint32_t *)d_pubkeys, n, strict, nullptr, results);
}

int ed25519_b200_verify_each_flat(dalek_b200_ctx *ctx, const uint8_t *msgs_flat, const uint64_t *msg_offsets, const uint8_t *sigs,
                                  const uint8_t *pubkeys, size_t n, int strict, uint8_t *results)
{
    if (!ctx || (n && (!sigs || !pubkeys || !results)) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    if ((rc = base_table_ensure(ctx))) return rc;
    if (ctx->opt_each_comb && ctx->opt_field_f64 && n) {
        // keys may repeat: everything crosses PCIe first (the key tables need every key), then either the comb path or,
        // when the keys turn out not to repeat, the plain kernel on the resident copies
        const size_t mbytes = (size_t)msg_offsets[n];
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], mbytes + 16))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_MSG_OFFSETS], (n + 1) * 8))) return rc;
        if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], n * 96))) return rc;
        uint8_t *d_msgs = (uint8_t *)ctx->ws[WS_STAGING_MSGS].p, *d_sigs = (uint8_t *)ctx->ws[WS_STAGING_IN].p, *d_keys = d_sigs + n * 64;
        uint64_t *d_offs = (uint64_t *)ctx->ws[WS_MSG_OFFSETS].p;
        cudaStream_t st = ctx->stream;
        if (mbytes) CUDA_TRY(ctx, cudaMemcpyAsync(d_msgs, msgs_flat, mbytes, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_offs, msg_offsets, (n + 1) * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_sigs, sigs, n * 64, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_keys, pubkeys, n * 32, cudaMemcpyHostToDevice, st));
        return verify_each_resident(ctx, d_msgs, d_offs, (const uint32_t *)d_sigs, (const uint32_t *)d_keys, n, strict, nullptr, results);
    }
    // independent per signature: pieces alternate between two streams (copy-in -> kernel -> copy-out)
    const ge_niels_packed *base = (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p;
    rc = run_pieces(ctx, msgs_flat, msg_offsets, sigs, 64, pubkeys, 32, results, 1, nullptr, 0, n,
                    [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *d_sigs, const uint8_t *d_keys, size_t m,
                        uint8_t *d_out, uint8_t *, cudaStream_t st) {
                        k_verify_each<<<cdiv(m, 128), 128, 0, st>>>(d_msgs, d_offs, (const uint32_t *)d_sigs, (const uint32_t *)d_keys,
                                                                    m, strict, base, d_out);
                        return 0;
                    });
    return rc ? rc : verify_each_summary(results, n);
}

// verify_prehashed[_strict] (verifying.rs:230-257, :424-459): both paths of verify_each on the resident copies of the
// inputs, with the challenge of Ed25519ph.  The prehashes have a fixed stride, so no offsets cross PCIe.
int ed25519_b200_verify_prehashed_each(dalek_b200_ctx *ctx, const uint8_t *prehashes, const uint8_t *context, size_t context_len,
                                       const uint8_t *sigs, const uint8_t *pubkeys, size_t n, int strict, uint8_t *results)
{
    if (!ctx || (n && (!prehashes || !sigs || !pubkeys || !results)) || (context_len && !context) || context_len > 255)
        return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    if (!n) return DALEK_OK;
    int rc;
    if ((rc = base_table_ensure(ctx))) return rc;
    Sha512Prefix dom;
    ed25519ph_dom2(dom, context, context_len);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], n * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], n * 96))) return rc;
    uint8_t *d_ph = (uint8_t *)ctx->ws[WS_STAGING_MSGS].p, *d_sigs = (uint8_t *)ctx->ws[WS_STAGING_IN].p, *d_keys = d_sigs + n * 64;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d_ph, prehashes, n * 64, cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_sigs, sigs, n * 64, cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_keys, pubkeys, n * 32, cudaMemcpyHostToDevice, st));
    return verify_each_resident(ctx, d_ph, nullptr, (const uint32_t *)d_sigs, (const uint32_t *)d_keys, n, strict, &dom, results);
}

}  // extern "C"

// ---- resident verifying-key sets ----------------------------------------------------------------------------------------
// A validator set, a service's known signers or a log's issuers are known before their signatures arrive.  A set
// decompresses and tabulates its k keys once (the per-key comb tables above, built by the same two kernels), keeps the 32
// bytes of each key as given (the challenge hashes VerifyingKey.compressed, the caller's encoding) and then verifies any
// number of calls through k_verify_each_comb, unchanged: a call hashes each signature under its key (k_key_set_front)
// and needs no key de-duplication, no table build and no host synchronisation before the comb kernel.
#define KEY_SET_BUILD_GROUP 4096        // keys per build pass: their 16^i A powers (WS_EACH_POW) stay at 40 MiB

struct ed25519_b200_key_set {
    dalek_b200_ctx *ctx;   // the context it serves; destroy does not touch it
    int device;
    size_t k;
    double *d_tab;         // k x EACH_KEY_DOUBLES: the comb tables k_verify_each_comb reads
    uint32_t *d_keys;      // k x 32 B as given, then k slot indices 0..k-1 (the `dense` map), then k status bytes
    uint32_t *d_slots;
    uint8_t *d_kstat;      // bit 0: the key did not decode, bit 1: small order (k_each_key_pow16)
};

// The workspace of a set call (WS_KEY_SET_FRONT): a status word (an index >= k was seen), then per signature h_i
// (32 B), the checked key index and the non-canonical-s mark.
struct KeySetFront { int *bad_idx; uint32_t *hs, *idx; uint8_t *bad_s; };

static int key_set_front_reserve(dalek_b200_ctx *ctx, size_t n, KeySetFront &f)
{
    int rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_KEY_SET_FRONT], 16 + n * 37))) return rc;
    char *p = (char *)ctx->ws[WS_KEY_SET_FRONT].p;
    f.bad_idx = (int *)p; f.hs = (uint32_t *)(p + 16); f.idx = f.hs + 8 * n; f.bad_s = (uint8_t *)(f.idx + n);
    CUDA_TRY(ctx, cudaMemsetAsync(f.bad_idx, 0, 4, ctx->stream));
    return 0;
}

// one thread per signature: the key index checked (an index >= k reads key 0 and sets *bad_idx), k = SHA-512(R || A ||
// M) mod l with A the set's stored bytes (PH = 1: SHA-512(dom2 || R || A || PH), prehash i at msgs + 64 i, offs unused;
// verifying.rs:515-535), and the canonical-s mark (signature.rs:89-94) -- what k_verify_each_comb reads
template <int PH>
__global__ void __launch_bounds__(128)
k_key_set_front(const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ offs, const __grid_constant__ Sha512Prefix dom,
                const uint32_t *__restrict__ sigs, const uint32_t *__restrict__ key_idx, size_t n, const uint32_t *__restrict__ keys,
                uint32_t k, uint32_t *__restrict__ hs, uint32_t *__restrict__ idx, uint8_t *__restrict__ bad_s, int *__restrict__ bad_idx)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t t = key_idx ? key_idx[i] : 0;
    if (t >= k) { t = 0; atomicOr(bad_idx, 1); }
    uint32_t R[8], s[8], A[8];
#pragma unroll
    for (int w = 0; w < 8; w++) { R[w] = sigs[16 * i + w]; s[w] = sigs[16 * i + 8 + w]; A[w] = keys[8 * (size_t)t + w]; }
    uint32_t dig[16], h[8];
    if (PH) sha512_pxm<2, 1>(dig, dom.b, dom.len, R, A, msgs + 64 * i, 64);
    else sha512_ram(dig, R, A, msgs + offs[i], (size_t)(offs[i + 1] - offs[i]));
    sc_reduce512(h, dig);
#pragma unroll
    for (int w = 0; w < 8; w++) hs[8 * i + w] = h[w];
    idx[i] = t;
    bad_s[i] = (uint8_t)!sc_is_canonical(s);
}

static int key_set_check(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s)
{
    if (!ctx || !s) return DALEK_E_INVALID_ARG;
    if (s->ctx != ctx) { ctx->last_error = "verifying-key set used with a context other than its own"; return DALEK_E_INVALID_ARG; }
    return 0;
}

// the comb kernel's shared-memory limit (once per context) and the table of B
static int key_set_prepare(dalek_b200_ctx *ctx)
{
    int rc;
    if ((rc = base_table_ensure(ctx))) return rc;
    if (!ctx->each_attr_set) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(k_verify_each_comb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EACH_COMB_SMEM));
        ctx->each_attr_set = true;
    }
    return 0;
}

// front + comb over m signatures (device inputs of this piece; the front arrays at f, item lo of the batch)
static void key_set_launch(const ed25519_b200_key_set *s, const uint8_t *d_msgs, const uint64_t *d_offs, const Sha512Prefix *ph_dom,
                           const uint32_t *d_sigs, const uint32_t *d_idx, size_t m, int strict, const KeySetFront &f, size_t lo,
                           const ge_niels_packed *base, uint8_t *d_out, cudaStream_t st)
{
    uint32_t *hs = f.hs + 8 * lo, *idx = f.idx + lo;
    uint8_t *bad_s = f.bad_s + lo;
    if (ph_dom)
        k_key_set_front<1><<<cdiv(m, 128), 128, 0, st>>>(d_msgs, nullptr, *ph_dom, d_sigs, d_idx, m, s->d_keys, (uint32_t)s->k, hs, idx,
                                                          bad_s, f.bad_idx);
    else
        k_key_set_front<0><<<cdiv(m, 128), 128, 0, st>>>(d_msgs, d_offs, Sha512Prefix{}, d_sigs, d_idx, m, s->d_keys, (uint32_t)s->k, hs,
                                                          idx, bad_s, f.bad_idx);
    k_verify_each_comb<<<cdiv((m + EACH_K - 1) / EACH_K, 128), 128, EACH_COMB_SMEM, st>>>(d_sigs, hs, bad_s, idx, s->d_slots, s->d_kstat,
                                                                                         s->d_tab, base, 0, m, strict, d_out);
}

// a whole batch whose inputs are in device memory (the _dev call, and the staged Ed25519ph call): both kernels, then
// the results and the index status read back
static int key_set_resident(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint8_t *d_msgs, const uint64_t *d_offs,
                            const Sha512Prefix *ph_dom, const uint32_t *d_sigs, const uint32_t *d_idx, size_t n, int strict,
                            uint8_t *results)
{
    int rc;
    KeySetFront f;
    if ((rc = key_set_prepare(ctx))) return rc;
    if ((rc = key_set_front_reserve(ctx, n, f))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_ITEM_STATUS], n))) return rc;
    if ((rc = pinned_reserve(ctx, 64))) return rc;
    uint8_t *d_out = (uint8_t *)ctx->ws[WS_ITEM_STATUS].p;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    key_set_launch(s, d_msgs, d_offs, ph_dom, d_sigs, d_idx, n, strict, f, 0, (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p, d_out, st);
    ctx->launches += 2;
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(results, d_out, n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_pinned, f.bad_idx, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = 2;
    if (*(const int *)ctx->h_pinned) { ctx->last_error = "key index >= len()"; return DALEK_E_INVALID_ARG; }
    return verify_each_summary(results, n);
}

static bool key_indices_ok(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint32_t *key_idx, size_t n)
{
    if (key_idx)                                                   // public: checked before any device work
        for (size_t i = 0; i < n; i++)
            if (key_idx[i] >= s->k) { ctx->last_error = "key index >= len()"; return false; }
    return true;
}

static void key_set_free(ed25519_b200_key_set *s)
{
    cudaFree(s->d_tab);                                            // waits for the device: no call still reads the set
    cudaFree(s->d_keys);
    delete s;
}

extern "C" {

int ed25519_b200_key_set_new(dalek_b200_ctx *ctx, const uint8_t *pubkeys, size_t k, uint8_t *ok, uint8_t *weak,
                             ed25519_b200_key_set **out)
{
    if (!ctx || !out) return DALEK_E_INVALID_ARG;
    *out = nullptr;
    if (!pubkeys || !k || k > 0xffffffffull) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CallTimer timer(ctx);
    int rc;
    const size_t group = std::min<size_t>(k, KEY_SET_BUILD_GROUP);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_EACH_POW], group * 64 * sizeof(ge_p3_raw)))) return rc;
    ed25519_b200_key_set *s = new (std::nothrow) ed25519_b200_key_set();
    uint32_t *slots = new (std::nothrow) uint32_t[k];
    uint8_t *kstat = new (std::nothrow) uint8_t[k];
    auto fail = [&](int code) {
        if (s) key_set_free(s);
        delete[] slots; delete[] kstat;
        return code;
    };
    if (!s || !slots || !kstat) { ctx->last_error = "out of host memory for the verifying-key set"; return fail(DALEK_E_NOMEM); }
    s->ctx = ctx; s->device = ctx->device; s->k = k;
    if (cudaMalloc((void **)&s->d_tab, k * EACH_KEY_DOUBLES * sizeof(double)) != cudaSuccess ||
        cudaMalloc((void **)&s->d_keys, k * (32 + 4 + 1)) != cudaSuccess) {
        (void)cudaGetLastError();
        ctx->last_error = "cudaMalloc failed for the verifying-key set";
        return fail(DALEK_E_NOMEM);
    }
    s->d_slots = s->d_keys + 8 * k;
    s->d_kstat = (uint8_t *)(s->d_slots + k);
    for (size_t i = 0; i < k; i++) slots[i] = (uint32_t)i;
    cudaStream_t st = ctx->stream;
    ge_p3_raw *pw = (ge_p3_raw *)ctx->ws[WS_EACH_POW].p;
    bool cuda_ok = cudaEventRecord(ctx->ev_a, st) == cudaSuccess &&
                   cudaMemcpyAsync(s->d_keys, pubkeys, k * 32, cudaMemcpyHostToDevice, st) == cudaSuccess &&
                   cudaMemcpyAsync(s->d_slots, slots, k * 4, cudaMemcpyHostToDevice, st) == cudaSuccess;
    for (size_t o = 0; cuda_ok && o < k; o += group) {             // uniq = slots 0..m-1 over the keys from o
        const size_t m = std::min(group, k - o);
        k_each_key_pow16<<<cdiv(m, 64), 64, 0, st>>>(s->d_keys + 8 * o, s->d_slots, m, pw, s->d_kstat + o);
        k_each_key_rows<<<cdiv(m * 512, 128), 128, 0, st>>>(pw, m, s->d_tab + o * EACH_KEY_DOUBLES);
        ctx->launches += 2;
        cuda_ok = cudaGetLastError() == cudaSuccess;
    }
    cuda_ok = cuda_ok && cudaEventRecord(ctx->ev_b, st) == cudaSuccess &&
              cudaMemcpyAsync(kstat, s->d_kstat, k, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
              cudaStreamSynchronize(st) == cudaSuccess;
    if (!cuda_ok) {
        ctx->last_error = std::string("verifying-key set build: ") + cudaGetErrorString(cudaGetLastError());
        return fail(DALEK_E_CUDA);
    }
    float ms = 0.f;
    if ((ms = elapsed_ms(ctx->ev_a, ctx->ev_b)) >= 0.f) ctx->last_kernel_ms = ms;
    ctx->last_kernel_launches = (int)(2 * ((k + group - 1) / group));
    bool all_ok = true;
    for (size_t i = 0; i < k; i++) {
        const bool good = !(kstat[i] & 1);
        all_ok &= good;
        if (ok) ok[i] = good;
        if (weak) weak[i] = good && (kstat[i] & 2);                // VerifyingKey::is_weak (verifying.rs:192-194)
    }
    if (!all_ok) { ctx->last_error = "a verifying key does not decode"; return fail(ED25519_ERR_POINT_DECOMPRESSION); }
    delete[] slots; delete[] kstat;
    *out = s;
    return DALEK_OK;
}

size_t ed25519_b200_key_set_len(const ed25519_b200_key_set *s) { return s ? s->k : 0; }

void ed25519_b200_key_set_destroy(ed25519_b200_key_set *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    key_set_free(s);
}

int ed25519_b200_key_set_verify_flat(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint8_t *msgs_flat,
                                     const uint64_t *msg_offsets, const uint8_t *sigs, const uint32_t *key_idx, size_t n,
                                     int strict, uint8_t *results)
{
    int rc;
    if ((rc = key_set_check(ctx, s))) return rc;
    if ((n && (!sigs || !results)) || !flat_messages_ok(msgs_flat, msg_offsets, n)) return DALEK_E_INVALID_ARG;
    if (!key_indices_ok(ctx, s, key_idx, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    KeySetFront f;
    if ((rc = key_set_prepare(ctx))) return rc;
    if ((rc = key_set_front_reserve(ctx, n, f))) return rc;
    const ge_niels_packed *base = (const ge_niels_packed *)ctx->ws[WS_BASE_TABLE].p;
    // independent per signature: pieces alternate between two streams (copy-in -> front + comb -> copy-out)
    rc = run_pieces(ctx, msgs_flat, msg_offsets, sigs, 64, (const uint8_t *)key_idx, key_idx ? 4 : 0, results, 1, nullptr, 0, n,
                    [&](const uint8_t *d_msgs, const uint64_t *d_offs, const uint8_t *d_sigs, const uint8_t *d_idx, size_t m,
                        uint8_t *d_out, uint8_t *, cudaStream_t st, size_t lo) {
                        key_set_launch(s, d_msgs, d_offs, nullptr, (const uint32_t *)d_sigs, key_idx ? (const uint32_t *)d_idx : nullptr,
                                       m, strict, f, lo, base, d_out, st);
                        ctx->launches++;                           // run_pieces counts one launch per piece
                        return 0;
                    });
    return rc ? rc : verify_each_summary(results, n);
}

int ed25519_b200_key_set_verify_flat_dev(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const void *d_msgs_flat,
                                         const void *d_msg_offsets, const void *d_sigs, const void *d_key_idx, size_t n, int strict,
                                         uint8_t *results)
{
    int rc;
    if ((rc = key_set_check(ctx, s))) return rc;
    if (n && (!d_msg_offsets || !d_sigs || !results)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    return key_set_resident(ctx, s, (const uint8_t *)d_msgs_flat, (const uint64_t *)d_msg_offsets, nullptr, (const uint32_t *)d_sigs,
                            (const uint32_t *)d_key_idx, n, strict, results);
}

// the three inputs have fixed widths, so they cross PCIe whole, as in verify_prehashed_each
int ed25519_b200_key_set_verify_prehashed(dalek_b200_ctx *ctx, const ed25519_b200_key_set *s, const uint8_t *prehashes,
                                          const uint8_t *context, size_t context_len, const uint8_t *sigs, const uint32_t *key_idx,
                                          size_t n, int strict, uint8_t *results)
{
    int rc;
    if ((rc = key_set_check(ctx, s))) return rc;
    if ((n && (!prehashes || !sigs || !results)) || (context_len && !context) || context_len > 255) return DALEK_E_INVALID_ARG;
    if (!key_indices_ok(ctx, s, key_idx, n)) return DALEK_E_INVALID_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (!n) return DALEK_OK;
    CallTimer timer(ctx);
    Sha512Prefix dom;
    ed25519ph_dom2(dom, context, context_len);
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_MSGS], n * 64))) return rc;
    if ((rc = ws_reserve(ctx, ctx->ws[WS_STAGING_IN], n * 68))) return rc;
    uint8_t *d_ph = (uint8_t *)ctx->ws[WS_STAGING_MSGS].p, *d_sigs = (uint8_t *)ctx->ws[WS_STAGING_IN].p, *d_idx = d_sigs + n * 64;
    cudaStream_t st = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d_ph, prehashes, n * 64, cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_sigs, sigs, n * 64, cudaMemcpyHostToDevice, st));
    if (key_idx) CUDA_TRY(ctx, cudaMemcpyAsync(d_idx, key_idx, n * 4, cudaMemcpyHostToDevice, st));
    return key_set_resident(ctx, s, d_ph, nullptr, &dom, (const uint32_t *)d_sigs, key_idx ? (const uint32_t *)d_idx : nullptr, n,
                            strict, results);
}

}  // extern "C"
