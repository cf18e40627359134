// Host emulation of one warp running the limb-parallel (20-lane) field and point code of warp4_f64.cuh -- squaring,
// inversion, extended addition, and the body of k_combine (Horner pass, encoding, limbs, is_identity) -- with the
// operand-rule assertions of the host field model switched on.  The emulated warp is the one of w4_host_check.cpp.
// TEST INFRASTRUCTURE (tests/test_w20_host.py): not a CPU fallback of the product.
#include "w4_host_check.cpp"

static void fe64_of(fe64 &o, const double *l) { for (int k = 0; k < 5; k++) o.v[k] = l[k]; }
static void fe64_bytes(uint32_t w[8], const fe64 &a) { fe f; fe64_to_fe(f, a); fe_tobytes_words(w, f); }

extern "C" {

// w20_sq and w20_invert on four elements (one per lane group) against fe64_sq / fe_invert, compared as canonical
// bytes.  a: 4 x 5 integer-valued limbs.  Returns 1 if all agree and every output limb is within scale 1.
int h_w20_sq_invert(const double *a)
{
    double sq[32], inv[32];
    run_warp([&](uint32_t lane) {
        const w20_role r = w20_roles();
        sq[lane] = w20_sq(a[5 * r.g + r.i], r);
        inv[lane] = w20_invert(a[5 * r.g + r.i], r);
    });
    for (int g = 0; g < 4; g++) {
        fe64 x, want, got_sq, got_inv;
        fe64_of(x, a + 5 * g);
        for (int k = 0; k < 5; k++) { got_sq.v[k] = sq[5 * g + k]; got_inv.v[k] = inv[5 * g + k]; }
        fe64_assert_scale(got_sq, 1.0); fe64_assert_scale(got_inv, 1.0);
        uint32_t bw[8], bg[8];
        fe64_sq(want, x);
        fe64_bytes(bw, want); fe64_bytes(bg, got_sq);
        if (memcmp(bw, bg, 32)) return 0;
        fe fx, fi; fe64_to_fe(fx, x); fe_invert(fi, fx); fe_tobytes_words(bw, fi);
        fe64_bytes(bg, got_inv);
        if (memcmp(bw, bg, 32)) return -2;
    }
    for (int l = 20; l < 32; l++) if (sq[l] != sq[l - 20] || inv[l] != inv[l - 20]) return -1;
    return 1;
}

// P + Q with w20_add (both points blinded to Z != 1) -> compressed
int h_w20_add(uint8_t *out, const uint8_t *ps, const uint8_t *qs)
{
    ge_p3 p, q, bp, bq;
    if (!load_point(p, ps) || !load_point(q, qs)) return 0;
    blind(bp, p); blind(bq, q);
    ge_p3_raw rp, rq; ge_p3_store_raw(rp, bp); ge_p3_store_raw(rq, bq);
    std::vector<uint8_t> outs(32 * 32);
    run_warp([&](uint32_t lane) {
        const w20_role r = w20_roles();
        fe64 d2v; fe64_const_2d(d2v);
        double c = w20_load(&rp, r);
        w20_add(c, w20_load(&rq, r), w20_limb(d2v, r.i), r);
        w4f_point t; w20_give(t, c);
        ge_p3 s; w4f_to_p3(s, t);
        store_point(&outs[32 * lane], s);
    });
    for (int l = 1; l < 32; l++) if (memcmp(&outs[0], &outs[32 * l], 32)) return -1;
    memcpy(out, &outs[0], 32);
    return 1;
}

// w20_load then w20_store (the raw points in and out of k_chunk_reduce / k_finish_windows): the same point back,
// with the very words the replicated form writes (w4f_load, fe64_to_fe, ge_p3_store_raw); returns -1 otherwise
int h_w20_store_roundtrip(uint8_t *out, const uint8_t *ps)
{
    ge_p3 p, bp; if (!load_point(p, ps)) return 0;
    blind(bp, p);
    ge_p3_raw rp, ro, want; ge_p3_store_raw(rp, bp);
    memset(&ro, 0xff, sizeof ro);
    run_warp([&](uint32_t) { const w20_role r = w20_roles(); w20_store(&ro, w20_load(&rp, r)); });
    w4f_point t; w4f_load(t, &rp);
    ge_p3 tp; w4f_to_p3(tp, t); ge_p3_store_raw(want, tp);
    if (memcmp(&ro, &want, sizeof ro)) return -1;
    ge_p3 q; ge_p3_load_raw(q, ro);
    store_point(out, q);
    return 1;
}

// The body of k_combine on the emulated warp: w20_horner, then w20_encode; s = encoding, limbs = fe_to_limbs51 of the
// projective total, *is_id = ge_is_identity.  Also runs the Horner pass in the replicated 4-lane form with w4f_add and
// the integer ge_compress; returns -3 if the two forms differ in any output (the encoding and every limb).
int h_w20_combine(uint8_t *s_out, uint64_t *limbs, uint32_t *is_id, const uint8_t *windows, int ranks, int nwin, int c)
{
    std::vector<ge_p3_raw> raw((size_t)ranks * nwin);
    for (int i = 0; i < ranks * nwin; i++) {
        ge_p3 p, q; if (!load_point(p, windows + 32 * i)) return 0;
        blind(q, p);
        ge_p3_store_raw(raw[i], q);
    }
    std::vector<uint32_t> enc(8 * 32);
    std::vector<uint64_t> lim(20 * 32);
    std::vector<uint32_t> idf(32);
    run_warp([&](uint32_t lane) {
        const w20_role r = w20_roles();
        ge_p3 P;
        w20_encode(&enc[8 * lane], P, w20_horner(raw.data(), ranks, nwin, c, r), r);
        uint64_t *l = &lim[20 * lane];
        fe_to_limbs51(l, P.X); fe_to_limbs51(l + 5, P.Y); fe_to_limbs51(l + 10, P.Z); fe_to_limbs51(l + 15, P.T);
        idf[lane] = ge_is_identity(P);
    });
    for (int l = 1; l < 32; l++)
        if (memcmp(&enc[0], &enc[8 * l], 32) || memcmp(&lim[0], &lim[20 * l], 160) || idf[0] != idf[l]) return -1;
    // the 4-lane form: w4f_add per window point, the doublings replicated, the integer inversion of ge_compress
    ge_p3 Q;
    run_warp([&](uint32_t lane) {
        const uint32_t role = lane & 3;
        fe64 d2; fe64_const_2d(d2);
        w4f_point tot, x; w4f_identity(tot);
        bool started = false;
        for (int w = nwin - 1; w >= 0; w--) {
            if (started) w20_dbl_n(tot, c);
            else {
                bool any = false;
                for (int k = 0; k < ranks; k++) { ge_p3 q; ge_p3_load_raw(q, raw[(size_t)k * nwin + w]); any |= !ge_is_identity(q); }
                if (!any) continue;
                started = true;
            }
            for (int k = 0; k < ranks; k++) { w4f_load(x, &raw[(size_t)k * nwin + w]); w4f_add(tot, x, d2, role); }
        }
        if (lane == 0) w4f_to_p3(Q, tot);
    });
    uint32_t s2[8]; ge_compress(s2, Q);
    uint64_t l2[20];
    fe_to_limbs51(l2, Q.X); fe_to_limbs51(l2 + 5, Q.Y); fe_to_limbs51(l2 + 10, Q.Z); fe_to_limbs51(l2 + 15, Q.T);
    if (memcmp(s2, &enc[0], 32) || memcmp(l2, &lim[0], 160) || ge_is_identity(Q) != idf[0]) return -3;
    memcpy(s_out, &enc[0], 32); memcpy(limbs, &lim[0], 160); *is_id = idf[0];
    return 1;
}

}  // extern "C"
