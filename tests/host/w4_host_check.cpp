// Host emulation of ONE WARP (32 host threads in lock step at every lane primitive) running the product's 4-lane
// FP64 point code -- warp4_f64.cuh (Horner pass of k_combine) and straus_vt.cuh (vartime Straus main loop, NAF,
// table of odd multiples) -- with the operand-rule assertions of the host field model switched on.
// TEST INFRASTRUCTURE (tests/test_fe_host.py): not a CPU fallback of the product.
#define FE_CHECK_BOUNDS 1
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <functional>
#include <vector>

#include "../../curve25519_dalek_b200/csrc/straus_vt.cuh"
#include "../../curve25519_dalek_b200/csrc/transcript_warp.cuh"

// ---- the emulated warp -------------------------------------------------------------------------------------------
static pthread_barrier_t g_bar;
static uint32_t g_slot[32];
static thread_local uint32_t t_lane;

uint32_t w4_lane() { return t_lane; }
uint32_t w4_shfl(uint32_t v, int src)
{
    g_slot[t_lane] = v;
    pthread_barrier_wait(&g_bar);
    uint32_t r = g_slot[src & 31];
    pthread_barrier_wait(&g_bar);
    return r;
}
uint32_t w4_shfl_down(uint32_t v, int delta)
{
    g_slot[t_lane] = v;
    pthread_barrier_wait(&g_bar);
    uint32_t src = t_lane + (uint32_t)delta;
    uint32_t r = src < 32 ? g_slot[src] : v;
    pthread_barrier_wait(&g_bar);
    return r;
}
bool w4_any(bool p)
{
    g_slot[t_lane] = p;
    pthread_barrier_wait(&g_bar);
    uint32_t r = 0;
    for (int i = 0; i < 32; i++) r |= g_slot[i];
    pthread_barrier_wait(&g_bar);
    return r != 0;
}

struct LaneArg { std::function<void(uint32_t)> *body; uint32_t lane; };
static void *lane_main(void *p) { LaneArg *a = (LaneArg *)p; t_lane = a->lane; (*a->body)(a->lane); return nullptr; }
static void run_warp(std::function<void(uint32_t)> body)
{
    pthread_barrier_init(&g_bar, nullptr, 32);
    pthread_t th[32]; LaneArg args[32];
    for (uint32_t l = 0; l < 32; l++) { args[l] = {&body, l}; pthread_create(&th[l], nullptr, lane_main, &args[l]); }
    for (uint32_t l = 0; l < 32; l++) pthread_join(th[l], nullptr);
    pthread_barrier_destroy(&g_bar);
}

// ---- helpers -----------------------------------------------------------------------------------------------------
static int load_point(ge_p3 &p, const uint8_t *s)
{
    uint32_t w[8]; memcpy(w, s, 32); fe x, y; if (!ge_decompress_affine(x, y, w)) return 0;
    p.X = x; p.Y = y; fe_1(p.Z); fe_mul(p.T, x, y); return 1;
}
static void store_point(uint8_t *s, const ge_p3 &p) { uint32_t w[8]; ge_compress(w, p); memcpy(s, w, 32); }
static void blind(ge_p3 &q, const ge_p3 &p) { ge_p3 d; ge_dbl(d, p); ge_add(q, d, p); ge_pniels n; ge_p3_to_pniels(n, d); ge_padd(q, q, n, 1); }   // same point, Z != 1

extern "C" {

// k_combine's Horner pass: windows = ranks x nwin compressed points (rank-major); out = compress(sum_w 2^(c w) sum_r W[r][w])
int h_w4f_horner(uint8_t *out, const uint8_t *windows, int ranks, int nwin, int c)
{
    std::vector<ge_p3_raw> raw((size_t)ranks * nwin);
    for (int i = 0; i < ranks * nwin; i++) {
        ge_p3 p, q; if (!load_point(p, windows + 32 * i)) return 0;
        blind(q, p);
        ge_p3_store_raw(raw[i], q);
    }
    std::vector<uint8_t> outs(32 * 32);
    run_warp([&](uint32_t lane) {
        w4f_point tot;
        w4f_horner(tot, raw.data(), ranks, nwin, c, lane & 3);
        ge_p3 total; w4f_to_p3(total, tot);
        store_point(&outs[32 * lane], total);
    });
    for (int l = 1; l < 32; l++) if (memcmp(&outs[0], &outs[32 * l], 32)) return -1;     // replicated in every lane
    memcpy(out, &outs[0], 32);
    return 1;
}

static int fe_is_xy_zt(const ge_p3 &p) { fe a, b; fe_mul(a, p.X, p.Y); fe_mul(b, p.Z, p.T); return fe_eq(a, b); }
static void store_coords(uint8_t *o, const ge_p3 &p)                    // canonical X | Y | Z | T, 32 bytes each
{
    const fe *c[4] = {&p.X, &p.Y, &p.Z, &p.T};
    for (int k = 0; k < 4; k++) { uint32_t w[8]; fe_tobytes_words(w, *c[k]); memcpy(o + 32 * k, w, 32); }
}

// The vartime Straus path of straus_vt.cu on ceil(n / 8) emulated warps: NAF, tables, per-warp loop, sum of the warps
// -> out (compressed).  groups (nullable): 8 * ceil(n / 8) records of 128 bytes, the accumulator of each group as
// straus_warp_accumulate leaves it, before the warp sum.  Returns 0 on an undecodable point, -1 if the lanes of a group
// disagree, -2 if a warp's sum (which the sum of the warps adds) has T != XY / Z.
int h_straus_groups(uint8_t *groups, uint8_t *out, const uint8_t *scalars, const uint8_t *points, int n)
{
    std::vector<int8_t> nafs((size_t)NAF_LEN * (n ? n : 1));
    std::vector<ge_pniels_packed> tables((size_t)8 * (n ? n : 1));
    for (int j = 0; j < n; j++) {
        uint32_t s[8]; memcpy(s, scalars + 32 * j, 32);
        naf5(&nafs[(size_t)NAF_LEN * j], s);
        ge_p3 p, q; if (!load_point(p, points + 32 * j)) return 0;
        blind(q, p);
        ge_pniels pn; ge_p3_to_pniels(pn, q);
        ge_pniels_packed pk; ge_pniels_pack(pk, pn);
        ge64_pniels pn64; ge64_pniels_unpack(pn64, pk);
        ge64_p3 A; ge64_identity(A);
        ge64_padd(A, A, pn64, 0u);                                     // as k_straus_prepare does
        straus_table5(&tables[(size_t)8 * j], A);
    }
    const int warps = (n + 7) / 8;
    ge_p3 total; ge_p3_identity(total);
    int rc = 1;
    for (int w = 0; w < warps; w++) {
        ge_p3 part;
        std::vector<uint8_t> acc(32 * 128);
        run_warp([&](uint32_t lane) {
            w4f_point Q;
            straus_warp_accumulate(Q, nafs.data(), tables.data(), (size_t)n, (size_t)w, lane & 3, lane >> 2);
            ge_p3 g; w4f_to_p3(g, Q);
            store_coords(&acc[128 * lane], g);
            straus_warp_sum(Q, lane & 3);
            if (lane == 0) w4f_to_p3(part, Q);
        });
        for (int l = 0; l < 32; l++) if (memcmp(&acc[128 * l], &acc[128 * (l & ~3)], 128)) rc = -1;
        if (groups) for (int g = 0; g < 8; g++) memcpy(groups + 128 * (8 * w + g), &acc[128 * 4 * g], 128);
        if (rc == 1 && !fe_is_xy_zt(part)) rc = -2;
        ge_add(total, total, part);
    }
    store_point(out, total);
    return rc;
}

int h_straus_vartime(uint8_t *out, const uint8_t *scalars, const uint8_t *points, int n) { return h_straus_groups(nullptr, out, scalars, points, n); }

// The 20-lane field multiplication (w20_mul: one limb per lane, transpose-sum by shuffles, one parallel round of carries)
// against the single-thread host model fe64_mul, compared as canonical bytes.  a, b: 4 x 5 limbs each (one element per lane
// group), integer-valued doubles chosen by the caller -- incl. the operand-rule extremes (|a_i b_j| just below 2^103).
// Returns 1 if all four products agree and every output limb is within scale 1.
int h_w20_mul(const double *a, const double *b)
{
    double out[32];
    run_warp([&](uint32_t lane) {
        const w20_role r = w20_roles();
        out[lane] = w20_mul(a[5 * r.g + r.i], b[5 * r.g + r.i], r);
    });
    for (int g = 0; g < 4; g++) {
        fe64 x, y, want, got;
        for (int k = 0; k < 5; k++) { x.v[k] = a[5 * g + k]; y.v[k] = b[5 * g + k]; got.v[k] = out[5 * g + k]; }
        fe64_mul(want, x, y);
        fe64_assert_scale(got, 1.0);
        fe fw, fg; fe64_to_fe(fw, want); fe64_to_fe(fg, got);
        uint32_t bw[8], bg[8]; fe_tobytes_words(bw, fw); fe_tobytes_words(bg, fg);
        if (memcmp(bw, bg, 32)) return 0;
    }
    for (int l = 20; l < 32; l++) if (out[l] != out[l - 20]) return -1;             // lanes 20..31 mirror lanes 0..11
    return 1;
}

// w20_carry (a limb-distributed fe64_carry) on four elements at once
int h_w20_carry(const double *a)
{
    double out[32];
    run_warp([&](uint32_t lane) { const w20_role r = w20_roles(); out[lane] = w20_carry(a[5 * r.g + r.i], r); });
    for (int g = 0; g < 4; g++) {
        fe64 x, want;
        for (int k = 0; k < 5; k++) x.v[k] = a[5 * g + k];
        fe64_carry(want, x);
        for (int k = 0; k < 5; k++) if (want.v[k] != out[5 * g + k]) return 0;
    }
    return 1;
}

// The raw output limbs of all 32 lanes of w20_mul (op 0), w20_carry (op 1) or w20_invert (op 2) for nw warps of four
// elements each (a, b: nw x 20 limbs as integers; out: nw x 32 limbs), so that the device build of the same code can be
// compared with this emulation limb for limb: the floored split, the carry rounded to nearest even, the carry schedule.
void h_w20_raw(int op, int nw, const long long *a, const long long *b, long long *out)
{
    run_warp([&](uint32_t lane) {
        const w20_role r = w20_roles();
        for (int w = 0; w < nw; w++) {
            const double x = (double)a[20 * w + r.base + r.i], y = (double)b[20 * w + r.base + r.i];
            const double o = op == 0 ? w20_mul(x, y, r) : op == 1 ? w20_carry(x, r) : w20_invert(x, r);
            out[32 * w + lane] = (long long)o;
        }
    });
}

// k doublings of one point on 20 lanes (w20_dbl_n) -> compressed
int h_w20_dbl_n(uint8_t *out, const uint8_t *point, int k)
{
    ge_p3 p, q; if (!load_point(p, point)) return 0;
    blind(q, p);
    ge_p3_raw raw; ge_p3_store_raw(raw, q);
    std::vector<uint8_t> outs(32 * 32);
    run_warp([&](uint32_t lane) {
        w4f_point t; w4f_load(t, &raw);
        w20_dbl_n(t, k);
        ge_p3 r; w4f_to_p3(r, t);
        store_point(&outs[32 * lane], r);
    });
    for (int l = 1; l < 32; l++) if (memcmp(&outs[0], &outs[32 * l], 32)) return -1;
    memcpy(out, &outs[0], 32);
    return 1;
}

// NAF digits of one scalar (NAF_LEN of them)
void h_naf5(int8_t *out, const uint8_t *scalar) { uint32_t s[8]; memcpy(s, scalar, 32); naf5(out, s); }

// one Merlin transcript of verify_batch on the emulated warp: hrams n x 64 B, sigs n x 64 B (R || s) -> zs n x 16 B
void h_merlin_zs(uint8_t *zs, const uint8_t *hrams, const uint8_t *sigs, uint64_t n)
{
    std::vector<uint32_t> h(16 * n), sg(16 * n), z(4 * n);
    memcpy(h.data(), hrams, 64 * n); memcpy(sg.data(), sigs, 64 * n);
    run_warp([&](uint32_t) { merlin_zs_warp(h.data(), sg.data(), n, z.data()); });
    memcpy(zs, z.data(), 16 * n);
}
// the constant prefix state and positions compiled into the product
void h_merlin_prefix(uint64_t *lanes25, uint32_t *pos, uint32_t *pos_begin)
{
    for (uint32_t l = 0; l < 25; l++) lanes25[l] = merlin_prefix_lane(l);
    *pos = MERLIN_PREFIX_POS; *pos_begin = MERLIN_PREFIX_POS_BEGIN;
}

}  // extern "C"
