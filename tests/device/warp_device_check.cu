// warp_device_check.cu -- TEST-ONLY kernels: run the product's lane-parallel point code (csrc/warp4.cuh, warp4_f64.cuh),
// the FP64 point formulas (csrc/ge64.cuh) and the FP64 exponentiation chains (csrc/fe64.cuh, x25519.cuh) on the device, on
// raw operands, and return the RAW output limbs of every lane, so that tests/test_gpu_warp_formulas.py can compare each
// output coordinate with exact integer formulas and check the limb bounds the headers state (a device build has no
// assertions).  Operands are free field elements, not points, so every limb can sit at its bound.
// Not part of libdalek_b200.so.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../curve25519_dalek_b200/csrc/warp4.cuh"
#include "../../curve25519_dalek_b200/csrc/warp4_f64.cuh"
#include "../../curve25519_dalek_b200/csrc/x25519.cuh"

__device__ __forceinline__ void ld64(fe64 &f, const long long *p) { for (int k = 0; k < 5; k++) f.v[k] = (double)p[k]; }
__device__ __forceinline__ void st64(long long *p, const fe64 &f) { for (int k = 0; k < 5; k++) p[k] = (long long)f.v[k]; }
__device__ __forceinline__ void ld_fe(fe &f, const long long *p) { for (int k = 0; k < 10; k++) f.v[k] = (uint32_t)p[k]; }
__device__ __forceinline__ void st_fe(long long *p, const fe &f) { for (int k = 0; k < 10; k++) p[k] = f.v[k]; }
__device__ __forceinline__ void ld_words(uint32_t *w, const long long *p, int n) { for (int k = 0; k < n; k++) w[k] = (uint32_t)p[k]; }
__device__ __forceinline__ void ld_bits(fe64 &f, const long long *p) { for (int k = 0; k < 5; k++) f.v[k] = __longlong_as_double(p[k]); }
__device__ __forceinline__ void st_bits(long long *p, const fe64 &f) { for (int k = 0; k < 5; k++) p[k] = __double_as_longlong(f.v[k]); }
__device__ __forceinline__ void ld_p64(w4f_point &p, const long long *s) { ld64(p.X, s); ld64(p.Y, s + 5); ld64(p.Z, s + 10); ld64(p.T, s + 15); }
__device__ __forceinline__ void st_p64(long long *d, const w4f_point &p) { st64(d, p.X); st64(d + 5, p.Y); st64(d + 10, p.Z); st64(d + 15, p.T); }
__device__ __forceinline__ void st_p32(uint32_t *d, const w4_point &p)
{
    for (int k = 0; k < 10; k++) { d[k] = p.X.v[k]; d[10 + k] = p.Y.v[k]; d[20 + k] = p.Z.v[k]; d[30 + k] = p.T.v[k]; }
}
__device__ __forceinline__ uint32_t warp_id() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }

// ---- 20-lane field: one warp per four elements, lane 5 g + i holds limb i of element g (lanes 20..31 mirror 0..11) ----
enum { W20_MUL = 0, W20_SQ = 1, W20_CARRY = 2, W20_SQN = 3, W20_INVERT = 4 };

// a, b: 20 limbs per warp; out: the limb of all 32 lanes
__global__ void k_w20_field(int op, uint32_t nw, const long long *a, const long long *b, int n, long long *out)
{
    const uint32_t w = warp_id();
    if (w >= nw) return;
    const w20_role r = w20_roles();
    const double x = (double)a[20 * w + r.base + r.i], y = (double)b[20 * w + r.base + r.i];
    double o;
    if (op == W20_MUL) o = w20_mul(x, y, r);
    else if (op == W20_SQ) o = w20_sq(x, r);
    else if (op == W20_CARRY) o = w20_carry(x, r);
    else if (op == W20_SQN) o = w20_sqn(x, n, r);
    else o = w20_invert(x, r);
    out[32 * w + w4_lane()] = (long long)o;
}

// ---- FP64 exponentiation chains and bit-pattern selects: one thread per element, 32 slots in and out ----------------
enum { CH_POW22501 = 0, CH_POW_P58 = 1, CH_INVERT_F64 = 2, CH_X25519_INVERT = 3, CH_FROMBYTES = 4, CH_CSWAP = 5, CH_CMOV = 6 };

__global__ void k_chain(int op, uint32_t n, const long long *in_, long long *out_)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const long long *in = in_ + 32 * (size_t)t;
    long long *out = out_ + 32 * (size_t)t;
    if (op == CH_POW22501) {                     // in: fe64 -> out: t19 | t3
        fe64 z, t19, t3; ld64(z, in); fe64_pow22501(t19, t3, z); st64(out, t19); st64(out + 5, t3);
    } else if (op == CH_POW_P58 || op == CH_INVERT_F64) {   // in: fe limbs -> out: fe limbs | canonical words
        fe f, h; ld_fe(f, in);
        if (op == CH_POW_P58) fe_pow_p58_f64(h, f); else fe_invert_f64(h, f);
        st_fe(out, h);
        uint32_t w[8]; fe_tobytes_words(w, h);
        for (int k = 0; k < 8; k++) out[10 + k] = w[k];
    } else if (op == CH_X25519_INVERT) {         // in: fe64 -> out: fe64
        fe64 z, r; ld64(z, in); x25519_invert(r, z); st64(out, r);
    } else if (op == CH_FROMBYTES) {             // in: 8 words -> out: limbs as read | after fe64_carry
        uint32_t w[8]; ld_words(w, in, 8);
        fe64 h, c; fe64_frombytes_words(h, w); fe64_carry(c, h); st64(out, h); st64(out + 5, c);
    } else if (op == CH_CSWAP) {                 // in: bits of a | bits of b | c -> out: a | b
        fe64 a, b; ld_bits(a, in); ld_bits(b, in + 5);
        fe64_cswap(a, b, (uint32_t)in[10]); st_bits(out, a); st_bits(out + 5, b);
    } else {                                     // CH_CMOV   in: bits of h | bits of g | c -> out: h
        fe64 h, g; ld_bits(h, in); ld_bits(g, in + 5);
        fe64_cmov(h, g, (uint32_t)in[10]); st_bits(out, h);
    }
}

// ---- FP64 point formulas, one thread per item -------------------------------------------------------------------------
// in (64 slots): p = X | Y | Z | T (fe64, 0..19); q at 20: affine Niels words (24), projective Niels words (32) or an
// extended fe64 point (20); neg at 60.   out (20 slots): X | Y | Z | T
enum { GE_MADD = 0, GE_PADD = 1, GE_DBL = 2, GE_DBL_NO_T = 3, GE_ADD_P3 = 4 };

__global__ void k_ge64(int op, uint32_t n, const long long *in_, long long *out_)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const long long *in = in_ + 64 * (size_t)t;
    ge64_p3 p, r;
    ld64(p.X, in); ld64(p.Y, in + 5); ld64(p.Z, in + 10); ld64(p.T, in + 15);
    fe64_0(r.X); fe64_0(r.Y); fe64_0(r.Z); fe64_0(r.T);
    const uint32_t neg = (uint32_t)in[60];
    if (op == GE_MADD) {
        ge_niels_packed pk; ld_words(pk.w, in + 20, 24);
        ge64_niels q; ge64_niels_unpack(q, pk); ge64_madd(r, p, q, neg);
    } else if (op == GE_PADD) {
        ge_pniels_packed pk; ld_words(pk.w, in + 20, 32);
        ge64_pniels q; ge64_pniels_unpack(q, pk); ge64_padd(r, p, q, neg);
    } else if (op == GE_DBL) ge64_dbl<true>(r, p);
    else if (op == GE_DBL_NO_T) ge64_dbl<false>(r, p);
    else {
        ge64_p3 q; ld64(q.X, in + 20); ld64(q.Y, in + 25); ld64(q.Z, in + 30); ld64(q.T, in + 35);
        fe64 d2; fe64_const_2d(d2); ge64_add_p3(r, p, q, d2);
    }
    long long *out = out_ + 20 * (size_t)t;
    st64(out, r.X); st64(out + 5, r.Y); st64(out + 10, r.Z); st64(out + 15, r.T);
}

// ---- 4-lane integer point code (warp4.cuh), one warp per item ------------------------------------------------------
// W4_ADD:   pts[2 item], pts[2 item + 1] -> p + q; every group stores its copy to st[8 item + group]
// W4_SHFL:  group g of warp `item` holds pts[8 item + g]; out = w4_shfl_down(., d)
// W4_FIXUP: the body of k_heavy_fixup on kk = arg task sums pts[(kk + 1) item + 1 ..], with the old sum pts[(kk + 1) item]
//           (first = 0) or the identity (first = 1); group 0 stores the result to st[8 item]
// out: the 40 limbs of every lane's point (X | Y | Z | T)
enum { W4_ADD = 0, W4_SHFL = 1, W4_FIXUP = 2 };

__global__ void k_w4(int op, uint32_t nw, const ge_p3_raw *pts, int arg, int first, uint32_t *out, ge_p3_raw *st)
{
    const uint32_t w = warp_id();
    if (w >= nw) return;
    const uint32_t lane = w4_lane(), role = lane & 3, grp = lane >> 2;
    w4_point acc, x;
    if (op == W4_ADD) {
        w4_load(acc, pts + 2 * w); w4_load(x, pts + 2 * w + 1);
        w4_add(acc, x, role);
        w4_store(st + 8 * w + grp, acc, role);
    } else if (op == W4_SHFL) {
        w4_load(x, pts + 8 * w + grp);
        w4_shfl_down(acc, x, arg);
    } else {
        const uint32_t kk = (uint32_t)arg;
        const ge_p3_raw *base = pts + (size_t)(kk + 1) * w;
        if (first || grp != 0) w4_identity(acc); else w4_load(acc, base);
        for (uint32_t j0 = 0; j0 < kk; j0 += 8) {
            const uint32_t j = j0 + grp;
            if (j < kk) w4_load(x, base + 1 + j); else w4_identity(x);
            w4_add(acc, x, role);
        }
        for (int d = 16; d >= 4; d >>= 1) { w4_shfl_down(x, acc, d); w4_add(acc, x, role); }
        if (grp == 0) w4_store(st + 8 * w, acc, role);
    }
    st_p32(out + 40 * (32 * (size_t)w + lane), acc);
}

// ---- 4-lane FP64 point code (warp4_f64.cuh), one warp per item; in: 64 slots per item as for k_ge64, d at 61 -------
// W4F_SHFL: group g of warp `item` holds the point of record 8 item + g.   out: the 20 limbs of every lane's point
enum { W4F_DBL = 0, W4F_ADD = 1, W4F_PADD = 2, W4F_SHFL = 3 };

__global__ void k_w4f(int op, uint32_t nw, const long long *in_, int arg, long long *out)
{
    const uint32_t w = warp_id();
    if (w >= nw) return;
    const uint32_t lane = w4_lane(), role = lane & 3, grp = lane >> 2;
    const long long *in = in_ + 64 * (size_t)w;
    w4f_point p, q;
    if (op == W4F_SHFL) {
        ld_p64(q, in_ + 64 * (8 * (size_t)w + grp));
        w4f_shfl_down(p, q, arg);
    } else {
        ld_p64(p, in);
        if (op == W4F_DBL) w4f_dbl(p, role, arg != 0);
        else if (op == W4F_ADD) { ld_p64(q, in + 20); fe64 d2; fe64_const_2d(d2); w4f_add(p, q, d2, role); }
        else { ge_pniels_packed pk; ld_words(pk.w, in + 20, 32); w4f_padd(p, pk, (uint32_t)in[60], role); }
    }
    st_p64(out + 20 * (32 * (size_t)w + lane), p);
}

// ---- 20-lane point code (warp4_f64.cuh), one warp per item -------------------------------------------------------
// W20_DBL / W20_ADD: in as for k_ge64 (p at 0, q at 20), lane 5 g + i takes limb i of coordinate g.
// W20_LOAD_STORE: c = w20_load(raw[item]), then w20_store(st + item, c).   out: the limb of all 32 lanes
enum { W20_DBL = 0, W20_ADD = 1, W20_LOAD_STORE = 2 };

__global__ void k_w20_point(int op, uint32_t nw, const long long *in_, const ge_p3_raw *raw, long long *out, ge_p3_raw *st)
{
    const uint32_t w = warp_id();
    if (w >= nw) return;
    const w20_role r = w20_roles();
    const long long *in = in_ + 64 * (size_t)w;
    double c;
    if (op == W20_DBL) { c = (double)in[r.base + r.i]; w20_dbl(c, r); }
    else if (op == W20_ADD) { c = (double)in[r.base + r.i]; w20_add(c, (double)in[20 + r.base + r.i], w20_const_2d(r), r); }
    else { c = w20_load(raw + w, r); w20_store(st + w, c); }
    out[32 * w + w4_lane()] = (long long)c;
}

// ---- the body of k_combine on one warp: w20_horner + w20_encode, and w4f_horner ------------------------------------
// out_s: every lane's encoding (8 words); out_p: every lane's point from w20_encode (40 limbs); out_tot: every lane's
// w4f_horner total (20 limbs)
__global__ void k_combine_body(const ge_p3_raw *windows, int ranks, int nwin, int c, uint32_t *out_s, uint32_t *out_p,
                               long long *out_tot)
{
    const uint32_t lane = w4_lane();
    const w20_role r = w20_roles();
    ge_p3 P;
    w20_encode(out_s + 8 * lane, P, w20_horner(windows, ranks, nwin, c, r), r);
    for (int k = 0; k < 10; k++) {
        out_p[40 * lane + k] = P.X.v[k]; out_p[40 * lane + 10 + k] = P.Y.v[k];
        out_p[40 * lane + 20 + k] = P.Z.v[k]; out_p[40 * lane + 30 + k] = P.T.v[k];
    }
    w4f_point tot;
    w4f_horner(tot, windows, ranks, nwin, c, lane & 3);
    st_p64(out_tot + 20 * lane, tot);
}

// ---- host side: copy in, launch, synchronise, copy out, return the CUDA status ----------------------------------------
struct DevBufs {
    void *p[4] = {nullptr, nullptr, nullptr, nullptr};
    ~DevBufs() { for (void *q : p) if (q) cudaFree(q); }
};

// buffers: in0 (copied in), in1 (copied in, optional), out0 and out1 (copied back, optional)
template <class F>
static int run(const void *in0, size_t b_in0, const void *in1, size_t b_in1, void *out0, size_t b_out0, void *out1,
               size_t b_out1, F launch)
{
    DevBufs d;
    const size_t sz[4] = {b_in0, b_in1, b_out0, b_out1};
    for (int k = 0; k < 4; k++)
        if (sz[k] && cudaMalloc(&d.p[k], sz[k]) != cudaSuccess) return (int)cudaGetLastError();
    cudaError_t e = cudaSuccess;
    if (b_in0) e = cudaMemcpy(d.p[0], in0, b_in0, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && b_in1) e = cudaMemcpy(d.p[1], in1, b_in1, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && b_out1) e = cudaMemset(d.p[3], 0xff, b_out1);
    if (e != cudaSuccess) return (int)e;
    launch(d.p[0], d.p[1], d.p[2], d.p[3]);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && b_out0) e = cudaMemcpy(out0, d.p[2], b_out0, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && b_out1) e = cudaMemcpy(out1, d.p[3], b_out1, cudaMemcpyDeviceToHost);
    return (int)e;
}

static unsigned warp_blocks(size_t nw) { return (unsigned)((nw + 3) / 4); }        // 4 warps per 128-thread block
static unsigned thread_blocks(size_t n) { return (unsigned)((n + 127) / 128); }

extern "C" {

// a, b: nw x 20 limbs; out: nw x 32 limbs
int w20_field_check(int op, size_t nw, const long long *a, const long long *b, int n, long long *out)
{
    return run(a, nw * 160, b ? b : a, nw * 160, out, nw * 256, nullptr, 0, [&](void *da, void *db, void *dout, void *) {
        k_w20_field<<<warp_blocks(nw), 128>>>(op, (uint32_t)nw, (const long long *)da, (const long long *)db, n, (long long *)dout);
    });
}

// in, out: n x 32 slots
int chain_check(int op, size_t n, const long long *in, long long *out)
{
    return run(in, n * 256, nullptr, 0, out, n * 256, nullptr, 0, [&](void *din, void *, void *dout, void *) {
        k_chain<<<thread_blocks(n), 128>>>(op, (uint32_t)n, (const long long *)din, (long long *)dout);
    });
}

// in: n x 64 slots; out: n x 20 limbs
int ge64_check(int op, size_t n, const long long *in, long long *out)
{
    return run(in, n * 512, nullptr, 0, out, n * 160, nullptr, 0, [&](void *din, void *, void *dout, void *) {
        k_ge64<<<thread_blocks(n), 128>>>(op, (uint32_t)n, (const long long *)din, (long long *)dout);
    });
}

// pts: npts raw points; out: nw x 32 x 40 limbs; st: nw x 8 raw points
int w4_check(int op, size_t nw, const void *pts, size_t npts, int arg, int first, uint32_t *out, void *st)
{
    return run(pts, npts * sizeof(ge_p3_raw), nullptr, 0, out, nw * 32 * 160, st, nw * 8 * sizeof(ge_p3_raw),
               [&](void *dp, void *, void *dout, void *dst) {
        k_w4<<<warp_blocks(nw), 128>>>(op, (uint32_t)nw, (const ge_p3_raw *)dp, arg, first, (uint32_t *)dout, (ge_p3_raw *)dst);
    });
}

// in: nrec x 64 slots (nw records, or 8 nw for W4F_SHFL); out: nw x 32 x 20 limbs
int w4f_check(int op, size_t nw, const long long *in, size_t nrec, int arg, long long *out)
{
    return run(in, nrec * 512, nullptr, 0, out, nw * 32 * 160, nullptr, 0, [&](void *din, void *, void *dout, void *) {
        k_w4f<<<warp_blocks(nw), 128>>>(op, (uint32_t)nw, (const long long *)din, arg, (long long *)dout);
    });
}

// in: nw x 64 slots (W20_DBL, W20_ADD) or raw: nw raw points (W20_LOAD_STORE); out: nw x 32 limbs; st: nw raw points
int w20_point_check(int op, size_t nw, const long long *in, const void *raw, long long *out, void *st)
{
    const bool ls = op == W20_LOAD_STORE;
    return run(ls ? raw : (const void *)in, nw * (ls ? sizeof(ge_p3_raw) : 512), nullptr, 0, out, nw * 256,
               ls ? st : nullptr, ls ? nw * sizeof(ge_p3_raw) : 0, [&](void *din, void *, void *dout, void *dst) {
        k_w20_point<<<warp_blocks(nw), 128>>>(op, (uint32_t)nw, (const long long *)din, (const ge_p3_raw *)din,
                                             (long long *)dout, (ge_p3_raw *)dst);
    });
}

// windows: ranks x nwin raw points (rank-major); out_s: 32 x 8 words; out_p: 32 x 40 limbs; out_tot: 32 x 20 limbs
int combine_check(const void *windows, int ranks, int nwin, int c, uint32_t *out_s, uint32_t *out_p, long long *out_tot)
{
    const size_t nb = (size_t)ranks * nwin * sizeof(ge_p3_raw);
    uint32_t *dsp = nullptr;
    if (cudaMalloc(&dsp, 32 * 48 * 4) != cudaSuccess) return (int)cudaGetLastError();
    int rc = run(windows, nb, nullptr, 0, out_tot, 32 * 160, nullptr, 0, [&](void *dw, void *, void *dt, void *) {
        k_combine_body<<<1, 32>>>((const ge_p3_raw *)dw, ranks, nwin, c, dsp, dsp + 32 * 8, (long long *)dt);
    });
    if (rc == 0) rc = (int)cudaMemcpy(out_s, dsp, 32 * 8 * 4, cudaMemcpyDeviceToHost);
    if (rc == 0) rc = (int)cudaMemcpy(out_p, dsp + 32 * 8, 32 * 40 * 4, cudaMemcpyDeviceToHost);
    cudaFree(dsp);
    return rc;
}

}  // extern "C"
