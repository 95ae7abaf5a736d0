// tests/hostsim/hostsim.cpp — TEST INFRASTRUCTURE: compiles the device math headers for the host
// (LHB_HOSTSIM: PTX carry chains emulated in C) so `-m "not gpu"` tests can check the exact limb algorithms
// against oracle/bls_ref.py without a GPU.  Never linked into liblhb200.so.
#define LHB_HOSTSIM 1
#include <string.h>
#include "../../lighthouse_b200/csrc/bls/fp.cuh"
#include "../../lighthouse_b200/csrc/bls/fp2.cuh"
#include "../../lighthouse_b200/csrc/bls/ec.cuh"
#include "../../lighthouse_b200/csrc/bls/h2c.cuh"
#include "../../lighthouse_b200/csrc/bls/pairing.cuh"
#include "../../lighthouse_b200/csrc/bls/miller_coop.cuh"
#include "../../lighthouse_b200/csrc/bls/miller_warp.cuh"
#include "../../lighthouse_b200/csrc/bls/g2_warp.cuh"
#include "../../lighthouse_b200/csrc/bls/fe_warp.cuh"
#include "../../lighthouse_b200/csrc/bls/fp_probe.cuh"
#include <vector>

using namespace lhb200::bls;
#define EXPORT extern "C" __attribute__((visibility("default")))

static void fp_in(Fp& r, const uint8_t* be48) { Fp c; fp_from_be48(c, be48); fp_to_mont(r, c); }
static void fp_out(uint8_t* be48, const Fp& a) { Fp c; fp_from_mont(c, a); fp_to_be48(be48, c); }
static void fp2_out(uint8_t* b, const Fp2& a) { fp_out(b, a.c0); fp_out(b + 48, a.c1); }
static void fp2_in(Fp2& r, const uint8_t* b) { fp_in(r.c0, b); fp_in(r.c1, b + 48); }

// op: 0 mul 1 add 2 sub 3 inv 4 neg 5 sqrt(returns ok)   (canonical big-endian 48-byte in/out)
EXPORT int hs_fp_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    Fp x, y, r; fp_in(x, a); fp_in(y, b);
    int ok = 1;
    switch (op) {
        case 0: fp_mul(r, x, y); break;
        case 1: fp_add(r, x, y); break;
        case 2: fp_sub(r, x, y); break;
        case 3: fp_inv(r, x); break;
        case 4: fp_neg(r, x); break;
        case 5: ok = fp_sqrt(r, x); break;
        case 6: fp_inv_vartime(r, x); break;
        default: return -1;
    }
    fp_out(out, r);
    return ok;
}
// raw Montgomery multiplication on little-endian limb arrays (no conversions): out = a*b/R mod p
EXPORT void hs_mont_mul_raw(const uint32_t* a, const uint32_t* b, uint32_t* out) {
    Fp x, y, r; memcpy(x.v, a, 48); memcpy(y.v, b, 48); fp_mul(r, x, y); memcpy(out, r.v, 48);
}
// op: 0 mul 1 sqr 2 inv 3 sqrt(ok) 4 sgn0
// split multiplier: redc(mulw(a, b)) in Montgomery limbs (raw)
EXPORT void hs_mont_mul_split(const uint32_t* a, const uint32_t* b, uint32_t* out) {
    Fp x, y, o; uint32_t w[24];
    for (int i = 0; i < 12; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
    fp_mulw_inl(w, x, y); fp_redc_inl(o, w);
    for (int i = 0; i < 12; i++) out[i] = o.v[i];
}
// dedicated squaring on raw Montgomery limbs
EXPORT void hs_mont_sqr(const uint32_t* a, uint32_t* out) {
    Fp x, o;
    for (int i = 0; i < 12; i++) x.v[i] = a[i];
    fp_sqr_inl(o, x);
    for (int i = 0; i < 12; i++) out[i] = o.v[i];
}
EXPORT int hs_fp2_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    Fp2 x, y, r; fp2_in(x, a); fp2_in(y, b);
    int ok = 1;
    switch (op) {
        case 0: fp2_mul(r, x, y); break;
        case 1: fp2_sqr(r, x); break;
        case 2: fp2_inv(r, x); break;
        case 3: ok = fp2_sqrt(r, x); break;
        case 4: ok = (int)fp2_sgn0(x); r = x; break;
        default: return -1;
    }
    fp2_out(out, r);
    return ok;
}
static void fp12_out(uint8_t* b, const Fp12& f) {
    const Fp2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
    for (int i = 0; i < 6; i++) fp2_out(b + 96 * i, *c[i]);
}
static void fp12_in(Fp12& f, const uint8_t* b) {
    Fp2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
    for (int i = 0; i < 6; i++) fp2_in(*c[i], b + 96 * i);
}
// op: 0 mul 1 sqr 2 inv 3 frob 4 frob2 5 cyclotomic_sqr 6 final_exp 7 mul_by_014 (b = c0|c1|c4 in first 3 fp2 slots)
EXPORT void hs_fp12_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
    Fp12 x, y, r; fp12_in(x, a); fp12_in(y, b);
    switch (op) {
        case 0: fp12_mul(r, x, y); break;
        case 1: fp12_sqr(r, x); break;
        case 2: fp12_inv(r, x); break;
        case 3: fp12_frob(r, x); break;
        case 4: fp12_frob2(r, x); break;
        case 5: fp12_cyclotomic_sqr(r, x); break;
        case 6: final_exp(r, x); break;
        case 7: fp12_mul_by_014(r, x, y.c0.c0, y.c0.c1, y.c0.c2); break;
    }
    fp12_out(out, r);
}
// G1: uncompressed 96 in -> [k]P uncompressed 96 out ; also compress/decompress
EXPORT int hs_g1_mul(const uint8_t* p96, const uint32_t* k, int nbits, uint8_t* out96, uint8_t* out48) {
    G1Affine a; if (g1_from_uncompressed(a, p96) == DEC_BAD) return -1;
    G1Jac j; jac_mul_affine(j, a, k, nbits);
    G1Affine r; jac_to_affine(r, j);
    g1_to_uncompressed(out96, r); g1_compress(out48, r);
    return 0;
}
EXPORT int hs_g1_decompress(const uint8_t* p48, uint8_t* out96) {
    G1Affine a; int rc = g1_decompress(a, p48); if (rc == DEC_BAD) return rc;
    g1_to_uncompressed(out96, a); return rc;
}
// sum of n uncompressed keys -> uncompressed
EXPORT int hs_g1_sum(const uint8_t* keys, int n, uint8_t* out96) {
    G1Jac acc; jac_set_inf(acc);
    for (int i = 0; i < n; i++) { G1Affine a; if (g1_from_uncompressed(a, keys + 96 * i) == DEC_BAD) return -1; jac_add_affine(acc, acc, a); }
    G1Affine r; jac_to_affine(r, acc); g1_to_uncompressed(out96, r); return 0;
}
// the device's 96-byte key decoding as lhb200_g1_deserialize_uncompressed applies it: g1_from_uncompressed, then the
// on-curve check for a finite point.  rc = DecodeStatus; out96 = the re-serialised point unless rc is DEC_BAD.
EXPORT int hs_g1_from_uncompressed(const uint8_t* p96, uint8_t* out96) {
    G1Affine a; int rc = g1_from_uncompressed(a, p96);
    if (rc == DEC_OK && !g1_on_curve(a)) rc = DEC_BAD;
    if (rc == DEC_BAD) return rc;
    g1_to_uncompressed(out96, a); return rc;
}
// bls/fp_probe.cuh on n cases (the body of lhb200_debug_fp_batch): in n x fp_probe_in_words(op), out n x 37 words.
// y operands are streamed at a stride of 3 words.  -1 for an unknown op.
EXPORT int hs_fp_batch(int op, const uint32_t* in, uint32_t n, uint32_t* out) {
    const int w = fp_probe_in_words(op);
    if (w == 0) return -1;
    std::vector<uint32_t> ycol(FP_PROBE_Y_WORDS * 3);
    for (uint32_t i = 0; i < n; i++) fp_probe(op, in + (size_t)w * i, ycol.data(), 3, out + (size_t)FP_PROBE_OUT_WORDS * i);
    return 0;
}
EXPORT int hs_g2_roundtrip(const uint8_t* p96, uint8_t* out96) {
    G2Affine a; int rc = g2_decompress(a, p96); if (rc == DEC_BAD) return rc;
    g2_compress(out96, a); return rc;
}
EXPORT int hs_g2_subgroup(const uint8_t* p96) {
    G2Affine a; int rc = g2_decompress(a, p96); if (rc == DEC_BAD) return -1;
    return g2_in_subgroup(a) ? 1 : 0;
}
EXPORT int hs_g1_subgroup(const uint8_t* p48) {
    G1Affine a; int rc = g1_decompress(a, p48); if (rc == DEC_BAD) return -1;
    return g1_in_subgroup(a) ? 1 : 0;
}
EXPORT int hs_g2_mul(const uint8_t* p96, const uint32_t* k, int nbits, uint8_t* out96) {
    G2Affine a; if (g2_decompress(a, p96) == DEC_BAD) return -1;
    G2Jac j; jac_mul_affine(j, a, k, nbits);
    G2Affine r; jac_to_affine(r, j); g2_compress(out96, r); return 0;
}
EXPORT void hs_hash_to_g2(const uint8_t* msg32, uint8_t* out96) {
    G2Jac j; hash_to_g2_jac(j, msg32);
    G2Affine r; jac_to_affine(r, j); g2_compress(out96, r);
}
EXPORT void hs_expand(const uint8_t* msg32, uint8_t* out256) { expand_message_xmd_256(msg32, out256); }
EXPORT void hs_sswu(const uint8_t* u96, uint8_t* xy192) {
    Fp2 u, x, y; fp2_in(u, u96); map_to_curve_sswu(x, y, u); fp2_out(xy192, x); fp2_out(xy192 + 96, y);
}
// miller loop (+ optional final exp) of (P uncompressed G1, Q compressed G2); proj: feed P as a re-randomised Jacobian
EXPORT int hs_pairing(const uint8_t* p96, const uint8_t* q96, int do_final, int proj, uint8_t* out576) {
    G1Affine p; G2Affine q;
    if (g1_from_uncompressed(p, p96) != DEC_OK || g2_decompress(q, q96) != DEC_OK) return -1;
    G1Proj3 pp;
    if (proj) {
        G1Jac j; jac_from_affine(j, p); jac_dbl(j, j);  // 2P in Jacobian form with Z != 1
        g1proj3_from_jac(pp, j);
    } else g1proj3_from_affine(pp, p);
    Fp12 f; miller_loop(f, pp, q);
    if (do_final) final_exp(f, f);
    fp12_out(out576, f);
    return 0;
}
// m pairs (P_j uncompressed G1, Q_j compressed G2).  The multi-pairing loop gets Q_j in Jacobian form with Z != 1
// (tripled and rescaled representative of the same point); out_multi = final_exp(miller_loop_multi),
// out_prod = final_exp(product of the single affine loops): equal although the raw Miller values differ by Fp2 factors.
EXPORT int hs_miller_multi(const uint8_t* p96, const uint8_t* q96, int m, uint8_t* out_multi, uint8_t* out_prod) {
    G1Proj3 P[MILLER_KMAX]; G2Affine Q[MILLER_KMAX]; G2Jac QJ[MILLER_KMAX]; uint32_t idx[MILLER_KMAX];
    if (m < 1 || m > MILLER_KMAX) return -2;
    for (int j = 0; j < m; j++) {
        G1Affine p;
        if (g1_from_uncompressed(p, p96 + 96 * j) != DEC_OK || g2_decompress(Q[j], q96 + 96 * j) != DEC_OK) return -1;
        G1Jac jj; jac_from_affine(jj, p); jac_dbl(jj, jj); g1proj3_from_jac(P[j], jj);
        // same point, non-trivial Z: (X s^2, Y s^3, s) with s taken from the point's own coordinates
        Fp2 s = Q[j].x, s2, s3; fp2_add(s, s, Q[j].y); fp2_sqr(s2, s); fp2_mul(s3, s2, s);
        fp2_mul(QJ[j].X, Q[j].x, s2); fp2_mul(QJ[j].Y, Q[j].y, s3); QJ[j].Z = s;
        idx[j] = (uint32_t)(m - 1 - j);  // permuted on purpose: the index list need not be sorted
    }
    Fp12 f, g, t;
    miller_loop_multi(f, P, QJ, idx, m);
    miller_loop(g, P[0], Q[0]);
    for (int j = 1; j < m; j++) { miller_loop(t, P[j], Q[j]); fp12_mul(g, g, t); }
    final_exp(f, f); final_exp(g, g);
    fp12_out(out_multi, f); fp12_out(out_prod, g);
    return 0;
}
// full single verification e(pk, H(m)) * e(-g1, sig) == 1
EXPORT int hs_verify(const uint8_t* pk96, const uint8_t* msg32, const uint8_t* sig96) {
    G1Affine pk, g1; G2Affine sig, h;
    if (g1_from_uncompressed(pk, pk96) != DEC_OK || g2_decompress(sig, sig96) != DEC_OK) return -1;
    if (!g2_in_subgroup(sig)) return -2;
    G2Jac hj; hash_to_g2_jac(hj, msg32); jac_to_affine(h, hj);
    g1.x = G1_GEN_X; fp_neg(g1.y, G1_GEN_Y); g1.inf = 0;
    G1Proj3 a, b; g1proj3_from_affine(a, pk); g1proj3_from_affine(b, g1);
    Fp12 f1, f2; miller_loop(f1, a, h); miller_loop(f2, b, sig);
    fp12_mul(f1, f1, f2); final_exp(f1, f1);
    return fp12_is_one(f1) ? 1 : 0;
}
EXPORT void hs_sswu_trace(const uint8_t* u96, uint8_t* out) {
    Fp2 u, x, y, tr[16]; fp2_in(u, u96); map_to_curve_sswu(x, y, u, tr);
    for (int k = 0; k < 16; k++) fp2_out(out + 96 * k, tr[k]);
}
EXPORT int hs_g2_mul_r_and_x(const uint8_t* p96, uint64_t r, uint8_t* out_r96, uint8_t* out_x96) {
    G2Affine a; if (g2_decompress(a, p96) == DEC_BAD) return -1;
    G2Jac jr, jx; g2_mul_r_and_x(jr, jx, a, r);
    G2Affine ar, ax; jac_to_affine(ar, jr); jac_to_affine(ax, jx);
    g2_compress(out_r96, ar); g2_compress(out_x96, ax); return 0;
}
EXPORT int hs_g1_mul_u64(const uint8_t* p96, uint64_t r, uint8_t* out96) {
    G1Affine a; if (g1_from_uncompressed(a, p96) == DEC_BAD) return -1;
    G1Jac j, o; jac_from_affine(j, a); jac_dbl(j, j);   // Jacobian base with Z != 1 (2P)
    jac_mul_u64(o, j, r);
    G1Affine ar; jac_to_affine(ar, o); g1_to_uncompressed(out96, ar); return 0;
}

// ---- fused sum-of-products Montgomery (bls/sop.cuh) on raw limbs: outA = sum_q xa_q ya_q / R, outB likewise (K = k <= 8).
// x operands as given (may be unreduced within the documented bounds); y operands streamed from a strided array.
template <int K>
static void hs_sop2_k(const uint32_t* xa, const uint32_t* ya, const uint32_t* xb, const uint32_t* yb, uint32_t* oa, uint32_t* ob) {
    const int stride = 3;   // deliberately not 1
    std::vector<uint32_t> ma(K * 12 * stride), mb(K * 12 * stride);
    SopX<K> XA, XB; SopY<K> YA, YB;
    YA.stride = stride; YB.stride = stride;
    for (int q = 0; q < K; q++) {
        for (int i = 0; i < 12; i++) {
            XA.x[q].v[i] = xa[12 * q + i]; XB.x[q].v[i] = xb[12 * q + i];
            ma[(q * 12 + i) * stride] = ya[12 * q + i]; mb[(q * 12 + i) * stride] = yb[12 * q + i];
        }
        YA.base[q] = &ma[q * 12 * stride]; YB.base[q] = &mb[q * 12 * stride];
    }
    Fp ra, rb;
    fp_sop2<K>(ra, rb, XA, YA, XB, YB);
    Fp r1;
    fp_sop1<K>(r1, XA, YA);
    for (int i = 0; i < 12; i++) { oa[i] = ra.v[i]; ob[i] = rb.v[i]; if (r1.v[i] != ra.v[i]) oa[i] = ~oa[i]; }
}
EXPORT int hs_sop2(int k, const uint32_t* xa, const uint32_t* ya, const uint32_t* xb, const uint32_t* yb, uint32_t* oa, uint32_t* ob) {
    switch (k) {
        case 1: hs_sop2_k<1>(xa, ya, xb, yb, oa, ob); return 0;
        case 2: hs_sop2_k<2>(xa, ya, xb, yb, oa, ob); return 0;
        case 4: hs_sop2_k<4>(xa, ya, xb, yb, oa, ob); return 0;
        case 6: hs_sop2_k<6>(xa, ya, xb, yb, oa, ob); return 0;
        case 8: hs_sop2_k<8>(xa, ya, xb, yb, oa, ob); return 0;
    }
    return -1;
}

// ---- the cooperative Miller program (bls/miller_coop.cuh) run lane by lane: NT = 14 lanes = 2 groups + 2 idle lanes per "warp".
// n pairs (P_j uncompressed G1 given as 2 P_j in projective form, Q_j compressed G2 handed over in Jacobian form with
// Z != 1); status[j] != 0 marks a set as skipped; with_extra appends (-g1, Q_extra).  Blocks of `spb` sets.
// out = final_exp(product of all group products) (576 bytes).
template <int NT>
struct ExecHost {
    std::vector<mc::Lane<NT>> lanes;
};
EXPORT int hs_miller_coop(const uint8_t* p96, const uint8_t* q96, const uint8_t* status, int n, const uint8_t* extra_q96,
                          int spb, uint8_t* out576) {
    constexpr int NT = 14;   // two working groups + two idle lanes (the device has 30 + 2)
    std::vector<G1Proj3> P(n); std::vector<G2Jac> H(n);
    for (int j = 0; j < n; j++) {
        G1Affine p; G2Affine q;
        if (g1_from_uncompressed(p, p96 + 96 * j) != DEC_OK) return -1;
        const int rc = g2_decompress(q, q96 + 96 * j);
        if (rc == DEC_BAD) return -1;
        G1Jac jj; jac_from_affine(jj, p); jac_dbl(jj, jj); g1proj3_from_jac(P[j], jj);
        if (rc == DEC_INFINITY) { jac_set_inf(H[j]); continue; }
        Fp2 s = q.x, s2, s3; fp2_add(s, s, q.y); fp2_sqr(s2, s); fp2_mul(s3, s2, s);
        fp2_mul(H[j].X, q.x, s2); fp2_mul(H[j].Y, q.y, s3); H[j].Z = s;
    }
    G2Jac extra; bool have_extra = extra_q96 != nullptr;
    if (have_extra) {
        G2Affine q; const int rc = g2_decompress(q, extra_q96);
        if (rc == DEC_BAD) return -1;
        if (rc == DEC_INFINITY) jac_set_inf(extra); else jac_from_affine(extra, q);
        G2Jac d; if (rc == DEC_OK) { jac_dbl(d, extra); jac_add(extra, d, extra); jac_neg(d, d); jac_add(extra, extra, d); }  // same point, Z != 1
    }
    const uint32_t n_total = n + (have_extra ? 1 : 0);
    const uint32_t n_blocks = (n_total + spb - 1) / spb;          // "warps" of NT lanes
    const uint32_t rounds_cap = (spb + NT - 1) / NT;
    std::vector<Fp12> outs(n_blocks);
    G1Proj3 neg_g1; neg_g1.px = G1_GEN_X; fp_neg(neg_g1.py, G1_GEN_Y); neg_g1.pz = FP_ONE;
    for (uint32_t b = 0; b < n_blocks; b++) {
        std::vector<uint32_t> smem(mc::region_words<NT>(), 0xdeadbeefu);
        std::vector<uint32_t> scratch((size_t)rounds_cap * 2 * mc::TWORDS * NT, 0xabababab);
        ExecHost<NT> ex;
        ex.lanes.resize(NT);
        for (int t = 0; t < NT; t++) {
            mc::Lane<NT>& L = ex.lanes[t];
            L.lane = t; L.t = t % 6; L.idle = t >= mc::lanes_used<NT>(); L.c = Col<NT>::make(smem.data(), t);
            L.act = reinterpret_cast<uint8_t*>(smem.data() + mc::NSLOT * NL * NT);
            L.active = false; L.extra = false; L.set = 0;
        }
        mc::Args a;
        a.P = P.data(); a.H = H.data(); a.status = status; a.n = n; a.extra_q = have_extra ? &extra : nullptr; a.extra_p = &neg_g1;
        a.lo = b * spb; a.hi = std::min<uint32_t>(n_total, a.lo + spb);
        a.scratch = scratch.data();
        mc::miller_program<NT>(ex, a);
        for (int t = 0; t < 6; t++) mc::store_group0(ex.lanes[t], outs[b]);
    }
    Fp12 f = outs[0];
    for (size_t i = 1; i < outs.size(); i++) fp12_mul(f, f, outs[i]);
    final_exp(f, f);
    fp12_out(out576, f);
    return 0;
}

// bls/miller_warp.cuh (one warp per pairing, Fp-granular phase tables), the 32 lanes of every phase run in sequence.
// Inputs as hs_miller_coop; `wpb` "warps" form a block whose values are multiplied by the dense section, like the kernel.
// out = final_exp(product of the block products).
EXPORT int hs_miller_warp(const uint8_t* p96, const uint8_t* q96, const uint8_t* status, int n, const uint8_t* extra_q96,
                          int wpb, uint8_t* out576) {
    std::vector<G1Proj3> P(n); std::vector<G2Jac> H(n);
    for (int j = 0; j < n; j++) {
        G1Affine p; G2Affine q;
        if (g1_from_uncompressed(p, p96 + 96 * j) != DEC_OK) return -1;
        const int rc = g2_decompress(q, q96 + 96 * j);
        if (rc == DEC_BAD) return -1;
        G1Jac jj; jac_from_affine(jj, p); jac_dbl(jj, jj); g1proj3_from_jac(P[j], jj);
        if (rc == DEC_INFINITY) { jac_set_inf(H[j]); continue; }
        Fp2 s = q.x, s2, s3; fp2_add(s, s, q.y); fp2_sqr(s2, s); fp2_mul(s3, s2, s);
        fp2_mul(H[j].X, q.x, s2); fp2_mul(H[j].Y, q.y, s3); H[j].Z = s;
    }
    G2Jac extra; const bool have_extra = extra_q96 != nullptr;
    if (have_extra) {
        G2Affine q; const int rc = g2_decompress(q, extra_q96);
        if (rc == DEC_BAD) return -1;
        if (rc == DEC_INFINITY) jac_set_inf(extra); else jac_from_affine(extra, q);
        G2Jac d; if (rc == DEC_OK) { jac_dbl(d, extra); jac_add(extra, d, extra); jac_neg(d, d); jac_add(extra, extra, d); }
    }
    G1Proj3 neg_g1; neg_g1.px = G1_GEN_X; fp_neg(neg_g1.py, G1_GEN_Y); neg_g1.pz = FP_ONE;
    const int n_total = n + (have_extra ? 1 : 0);
    const mw::Tables T = mw::miller_tables();
    Fp12 f; bool have_f = false;
    for (int b0 = 0; b0 < n_total; b0 += wpb) {
        std::vector<std::vector<uint32_t>> R(wpb, std::vector<uint32_t>(mw::REGION_WORDS, 0xdeadbeefu));
        for (int wib = 0; wib < wpb; wib++) {
            uint32_t* r = R[wib].data();
            for (int w = 0; w < 24 * mw::SL; w++) mw::set_one_words(r, w);
            const int set = b0 + wib;
            if (set >= n_total) continue;
            const G2Jac* q; const G1Proj3* p;
            if (set >= n) { q = &extra; p = &neg_g1; } else { q = &H[set]; p = &P[set]; if (status[set]) continue; }
            if (jac_is_inf(*q)) continue;
            const uint32_t* qs = reinterpret_cast<const uint32_t*>(q);
            for (int w = 0; w < 6 * NL; w++) r[(mw::MW_S_HX_0 + w / NL) * mw::SL + w % NL] = qs[w];
            const uint32_t* ps = reinterpret_cast<const uint32_t*>(p);
            for (int w = 0; w < 3 * NL; w++) r[(mw::MW_S_PX + w / NL) * mw::SL + w % NL] = ps[w];
            using namespace mw;
            MW_RUN(r, 0, INIT);
            for (int i = 62; i >= 0; i--) {
                MW_RUN(r, 0, SQR);
                MW_RUN(r, 0, DBL);
                MW_RUN(r, 0, SPARSE);
                if ((BLS_X_ABS >> i) & 1) {
                    MW_RUN(r, 0, ADD);
                    MW_RUN(r, 0, SPARSE);
                }
            }
            MW_RUN(r, 0, CONJ);
        }
        for (int stride = 1; stride < wpb; stride *= 2)
            for (int wib = 0; wib + stride < wpb; wib += 2 * stride) {
                uint32_t* r = R[wib].data(); const uint32_t* o = R[wib + stride].data();
                for (int w = 0; w < 24 * mw::SL; w++) r[mw::MW_S_G0_0 * mw::SL + w] = o[mw::MW_S_F0_0 * mw::SL + w];
                using namespace mw;
                MW_RUN(r, 0, DENSE);
            }
        Fp12 blk;
        uint32_t* o = reinterpret_cast<uint32_t*>(&blk);
        for (int w = 0; w < 12 * NL; w++) {
            const int fp2_idx = w / (2 * NL), comp = (w / NL) & 1, limb = w % NL;
            const int k = fp2_idx < 3 ? 2 * fp2_idx : 2 * (fp2_idx - 3) + 1;
            o[w] = R[0][(mw::MW_S_F0_0 + 4 * k + comp) * mw::SL + limb];
        }
        if (have_f) fp12_mul(f, f, blk); else { f = blk; have_f = true; }
    }
    final_exp(f, f);
    fp12_out(out576, f);
    return 0;
}

// bls/g2_warp.cuh, lane by lane: the signature program (r * sig, subgroup test) and clear_cofactor.
// hs_sig_warp: rc -1 bad encoding, 0 not in G2, 1 in G2 (out96 = compressed [r] sig).
EXPORT int hs_sig_warp(const uint8_t* sig96, uint64_t r, uint8_t* out96) {
    using namespace gw;
    G2Affine a;
    if (g2_decompress(a, sig96) != DEC_OK) return -1;
    std::vector<uint32_t> Rv(REGION_WORDS, 0xdeadbeefu);
    uint32_t* R = Rv.data();
    const mw::Tables T = tables();
    put_consts(R);
    put_fp2(R, GW_S_BPX_0, a.x); put_fp2(R, GW_S_BPX_0 + 2, a.y);
    Fp2 one; fp2_set_one(one); put_fp2(R, GW_S_BPX_0 + 4, one);
    GW_RUN(R, 0, SETA);
    GW_LADDER(R, 0, r, true, BLS_X_ABS);
    GW_RUN(R, 0, SIGCHECK);
    if (!(slots_zero(R, GW_S_E1_0, 4) && !slots_zero(R, GW_S_A2X_0 + 4, 2))) return 0;
    GW_RUN(R, 0, TOJAC);
    G2Jac j; get_fp2(j.X, R, GW_S_JX_0); get_fp2(j.Y, R, GW_S_JX_0 + 2); get_fp2(j.Z, R, GW_S_JX_0 + 4);
    G2Affine o; jac_to_affine(o, j); g2_compress(out96, o);
    return 1;
}
// out96 = compressed clear_cofactor(P) for the curve point P (compressed, not necessarily in G2)
EXPORT int hs_clear_cofactor_warp(const uint8_t* p96, uint8_t* out96) {
    using namespace gw;
    G2Affine a;
    if (g2_decompress(a, p96) != DEC_OK) return -1;
    G2Jac h; jac_from_affine(h, a); jac_dbl(h, h); G2Jac a2; jac_from_affine(a2, a); jac_neg(a2, a2); jac_add(h, h, a2);  // P with Z != 1
    std::vector<uint32_t> Rv(REGION_WORDS, 0xdeadbeefu);
    uint32_t* R = Rv.data();
    const mw::Tables T = tables();
    put_consts(R);
    put_fp2(R, GW_S_HX_0, h.X); put_fp2(R, GW_S_HX_0 + 2, h.Y); put_fp2(R, GW_S_HX_0 + 4, h.Z);
    GW_CLEAR_COFACTOR(R, 0);
    G2Jac j; get_fp2(j.X, R, GW_S_JX_0); get_fp2(j.Y, R, GW_S_JX_0 + 2); get_fp2(j.Z, R, GW_S_JX_0 + 4);
    G2Affine o; jac_to_affine(o, j); g2_compress(out96, o);
    return 0;
}

// bls/fe_warp.cuh lane by lane: out = final exponentiation of a * b (the product section folds the inputs), 576 bytes each
EXPORT int hs_final_warp(const uint8_t* a576, const uint8_t* b576, uint8_t* out576) {
    using namespace fe;
    Fp12 a, b2; fp12_in(a, a576); fp12_in(b2, b576);
    std::vector<uint32_t> Rv(REGION_WORDS, 0xdeadbeefu);
    uint32_t* R = Rv.data();
    const mw::Tables T = tables();
    const uint32_t* aw = reinterpret_cast<const uint32_t*>(&a); const uint32_t* bw = reinterpret_cast<const uint32_t*>(&b2);
    for (int w = 0; w < 12 * NL; w++) { R[reg_word(FE_S_F0_0, w)] = aw[w]; R[reg_word(FE_S_T00_0, w)] = bw[w]; }
    FE_RUN(R, 0, MUL_F_F_T0);
    Fp12 f, inv; uint32_t* fw = reinterpret_cast<uint32_t*>(&f);
    for (int w = 0; w < 12 * NL; w++) fw[w] = R[reg_word(FE_S_F0_0, w)];
    fp12_inv(inv, f);
    put_consts(R);
    const uint32_t* iw = reinterpret_cast<const uint32_t*>(&inv);
    for (int w = 0; w < 12 * NL; w++) R[reg_word(FE_S_T10_0, w)] = iw[w];
    FE_AFTER_INVERSION(R, 0);
    Fp12 g; uint32_t* gw_ = reinterpret_cast<uint32_t*>(&g);
    for (int w = 0; w < 12 * NL; w++) gw_[w] = R[reg_word(FE_S_F0_0, w)];
    fp12_out(out576, g);
    return 0;
}

// the sum tree step of k_g2_sum_warp lane by lane: sum of n compressed G2 points (infinity encodings skipped), each fed as a
// Jacobian point with Z != 1; out96 = compressed sum (the infinity encoding if nothing was added)
EXPORT int hs_g2_sum_warp(const uint8_t* pts96, int n, uint8_t* out96) {
    using namespace gw;
    std::vector<uint32_t> Rv(REGION_WORDS, 0xdeadbeefu);
    uint32_t* R = Rv.data();
    const mw::Tables T = tables();
    put_consts(R);
    bool have = false;
    for (int j = 0; j < n; j++) {
        G2Affine a; const int rc = g2_decompress(a, pts96 + 96 * j);
        if (rc == DEC_BAD) return -1;
        if (rc == DEC_INFINITY) continue;
        G2Jac h; jac_from_affine(h, a); jac_dbl(h, h); G2Jac na; jac_from_affine(na, a); jac_neg(na, na); jac_add(h, h, na);   // same point, Z != 1
        put_fp2(R, GW_S_HX_0, h.X); put_fp2(R, GW_S_HX_0 + 2, h.Y); put_fp2(R, GW_S_HX_0 + 4, h.Z);
        if (!have) { GW_RUN(R, 0, HINIT); have = true; }
        else { GW_RUN(R, 0, HBP); GW_RUN(R, 0, ADDA); }
    }
    G2Affine o;
    if (have) {
        GW_RUN(R, 0, TOJAC);
        G2Jac jj; get_fp2(jj.X, R, GW_S_JX_0); get_fp2(jj.Y, R, GW_S_JX_0 + 2); get_fp2(jj.Z, R, GW_S_JX_0 + 4);
        jac_to_affine(o, jj);
    } else { f_set_zero(o.x); f_set_zero(o.y); o.inf = 1; }
    g2_compress(out96, o);
    return 0;
}
