/*
 * oracle/bls12_381.c — TEST INFRASTRUCTURE ONLY (CPU oracle for bulk checks + the timed CPU baseline).
 *
 * Plain-C (6 x 64-bit limbs, unsigned __int128) restatement of the batch BLS verification path of
 * sigp/lighthouse v5.3.0: bls::verify_signature_sets (crypto/bls/src/impls/blst.rs:37-119) with the semantics of
 * SURVEY.md Appendix C.  The arithmetic itself lives in blst 0.3.12 (Cargo.lock:1023, not vendored): the
 * published algorithms (IETF BLS signatures, POP ciphersuite; RFC 9380 hash_to_curve for BLS12381G2_XMD:SHA-256_SSWU_RO_;
 * optimal-ate pairing) are restated here.  Work is spread over host threads the way blst's pool does
 * (block_signature_verifier.rs:413-414): per-thread Miller-loop products and signature sums, one merge, one
 * final exponentiation.
 *
 * Pinned by tests/test_oracle_bls.py: bit-exact against oracle/bls_ref.py (itself pinned by the reference's 22
 * deposit vectors and 10 interop key pairs) on hash_to_g2, aggregation, pairing values and batch verdicts.
 * Nothing in lighthouse_b200/ links or calls this file.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))
typedef unsigned __int128 u128;
typedef struct { uint64_t l[6]; } fp;
typedef struct { fp c0, c1; } fp2;
typedef struct { fp2 c0, c1, c2; } fp6;
typedef struct { fp6 c0, c1; } fp12;
#include "bls_consts64.h"

void orc_sha256(const uint8_t *msg, uint64_t len, uint8_t out[32]);   /* ssz_sha256.c */
typedef void (*range_fn)(uint64_t lo, uint64_t hi, void *ctx);
void orc_par_for(uint64_t n, uint64_t min_grain, range_fn fn, void *ctx);
int orc_num_threads(void);

static __thread uint64_t g_mulcount; /* instrumented Fp-multiplication counter (SURVEY §8d) */

/* ------------------------------------------------------------------------------------------------ Fp */
static inline int fp_is_zero(const fp *a) { return (a->l[0] | a->l[1] | a->l[2] | a->l[3] | a->l[4] | a->l[5]) == 0; }
static inline int fp_eq(const fp *a, const fp *b) {
    uint64_t o = 0;
    for (int i = 0; i < 6; i++) o |= a->l[i] ^ b->l[i];
    return o == 0;
}
static inline void fp_cond_sub(fp *r, const uint64_t t[6], uint64_t top) {
    uint64_t s[6], brw = 0;
    for (int i = 0; i < 6; i++) {
        u128 d = (u128)t[i] - C_P.l[i] - brw;
        s[i] = (uint64_t)d;
        brw = (uint64_t)(d >> 64) & 1;
    }
    int keep = (top == 0) && brw;
    for (int i = 0; i < 6; i++) r->l[i] = keep ? t[i] : s[i];
}
static inline void fp_add(fp *r, const fp *a, const fp *b) {
    uint64_t t[6], c = 0;
    for (int i = 0; i < 6; i++) {
        u128 s = (u128)a->l[i] + b->l[i] + c;
        t[i] = (uint64_t)s;
        c = (uint64_t)(s >> 64);
    }
    fp_cond_sub(r, t, c);
}
static inline void fp_sub(fp *r, const fp *a, const fp *b) {
    uint64_t t[6], brw = 0;
    for (int i = 0; i < 6; i++) {
        u128 d = (u128)a->l[i] - b->l[i] - brw;
        t[i] = (uint64_t)d;
        brw = (uint64_t)(d >> 64) & 1;
    }
    uint64_t m = 0 - brw, c = 0;
    for (int i = 0; i < 6; i++) {
        u128 s = (u128)t[i] + (C_P.l[i] & m) + c;
        r->l[i] = (uint64_t)s;
        c = (uint64_t)(s >> 64);
    }
}
static inline void fp_neg(fp *r, const fp *a) {
    fp z = {{0, 0, 0, 0, 0, 0}};
    fp_sub(r, &z, a);
}
static void fp_mul(fp *r, const fp *a, const fp *b) {
    g_mulcount++;
    uint64_t t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 6; i++) {
        uint64_t c = 0;
        for (int j = 0; j < 6; j++) {
            u128 acc = (u128)a->l[j] * b->l[i] + t[j] + c;
            t[j] = (uint64_t)acc;
            c = (uint64_t)(acc >> 64);
        }
        u128 acc = (u128)t[6] + c;
        t[6] = (uint64_t)acc;
        t[7] = (uint64_t)(acc >> 64);
        uint64_t m = t[0] * C_N0;
        acc = (u128)m * C_P.l[0] + t[0];
        c = (uint64_t)(acc >> 64);
        for (int j = 1; j < 6; j++) {
            acc = (u128)m * C_P.l[j] + t[j] + c;
            t[j - 1] = (uint64_t)acc;
            c = (uint64_t)(acc >> 64);
        }
        acc = (u128)t[6] + c;
        t[5] = (uint64_t)acc;
        t[6] = t[7] + (uint64_t)(acc >> 64);
    }
    fp_cond_sub(r, t, t[6]);
}
static inline void fp_sqr(fp *r, const fp *a) { fp_mul(r, a, a); }
/* a^((p-3)/4), 4-bit windows */
static void fp_pow_pm3d4(fp *r, const fp *a) {
    fp tab[16], acc;
    tab[1] = *a;
    for (int i = 2; i < 16; i++) fp_mul(&tab[i], &tab[i - 1], a);
    int started = 0;
    for (int w = 95; w >= 0; w--) {
        int bit = 4 * w;
        unsigned d = (unsigned)(C_EXP_PM3D4[bit >> 6] >> (bit & 63)) & 15u;
        if (started) {
            fp_sqr(&acc, &acc); fp_sqr(&acc, &acc); fp_sqr(&acc, &acc); fp_sqr(&acc, &acc);
            if (d) fp_mul(&acc, &acc, &tab[d]);
        } else if (d) { acc = tab[d]; started = 1; }
    }
    *r = acc;
}
static void fp_inv(fp *r, const fp *a) {
    fp t;
    fp_pow_pm3d4(&t, a);
    fp_sqr(&t, &t); fp_sqr(&t, &t);
    fp_mul(r, &t, a);
}
static int fp_sqrt(fp *r, const fp *a) {
    fp t, c;
    fp_pow_pm3d4(&t, a);
    fp_mul(&t, &t, a);
    fp_sqr(&c, &t);
    *r = t;
    return fp_eq(&c, a);
}
static void fp_from_mont(fp *r, const fp *a) { fp one = {{1, 0, 0, 0, 0, 0}}; fp_mul(r, a, &one); }
static void fp_to_mont(fp *r, const fp *a) { fp_mul(r, a, &C_R2); }
static void fp_from_be48(fp *c, const uint8_t *b) {
    for (int i = 0; i < 6; i++) {
        uint64_t v = 0;
        for (int k = 0; k < 8; k++) v = (v << 8) | b[8 * (5 - i) + k];
        c->l[i] = v;
    }
}
static void fp_to_be48(uint8_t *b, const fp *c) {
    for (int i = 0; i < 6; i++)
        for (int k = 0; k < 8; k++) b[8 * (5 - i) + k] = (uint8_t)(c->l[i] >> (56 - 8 * k));
}
static int fp_canon_cmp(const fp *a, const fp *b) { /* -1,0,1 */
    for (int i = 5; i >= 0; i--)
        if (a->l[i] != b->l[i]) return a->l[i] > b->l[i] ? 1 : -1;
    return 0;
}

/* ------------------------------------------------------------------------------------------------ Fp2 */
static inline void fp2_add(fp2 *r, const fp2 *a, const fp2 *b) { fp_add(&r->c0, &a->c0, &b->c0); fp_add(&r->c1, &a->c1, &b->c1); }
static inline void fp2_sub(fp2 *r, const fp2 *a, const fp2 *b) { fp_sub(&r->c0, &a->c0, &b->c0); fp_sub(&r->c1, &a->c1, &b->c1); }
static inline void fp2_neg(fp2 *r, const fp2 *a) { fp_neg(&r->c0, &a->c0); fp_neg(&r->c1, &a->c1); }
static inline void fp2_conj(fp2 *r, const fp2 *a) { r->c0 = a->c0; fp_neg(&r->c1, &a->c1); }
static inline void fp2_dbl(fp2 *r, const fp2 *a) { fp2_add(r, a, a); }
static inline int fp2_is_zero(const fp2 *a) { return fp_is_zero(&a->c0) && fp_is_zero(&a->c1); }
static inline int fp2_eq(const fp2 *a, const fp2 *b) { return fp_eq(&a->c0, &b->c0) && fp_eq(&a->c1, &b->c1); }
static void fp2_mul(fp2 *r, const fp2 *a, const fp2 *b) {
    fp t0, t1, s0, s1;
    fp_mul(&t0, &a->c0, &b->c0);
    fp_mul(&t1, &a->c1, &b->c1);
    fp_add(&s0, &a->c0, &a->c1);
    fp_add(&s1, &b->c0, &b->c1);
    fp_mul(&s0, &s0, &s1);
    fp_sub(&r->c0, &t0, &t1);
    fp_sub(&s0, &s0, &t0);
    fp_sub(&r->c1, &s0, &t1);
}
static void fp2_sqr(fp2 *r, const fp2 *a) {
    fp s, d, m;
    fp_add(&s, &a->c0, &a->c1);
    fp_sub(&d, &a->c0, &a->c1);
    fp_mul(&m, &a->c0, &a->c1);
    fp_mul(&r->c0, &s, &d);
    fp_add(&r->c1, &m, &m);
}
static inline void fp2_mul_fp(fp2 *r, const fp2 *a, const fp *s) { fp_mul(&r->c0, &a->c0, s); fp_mul(&r->c1, &a->c1, s); }
static inline void fp2_mul_xi(fp2 *r, const fp2 *a) {
    fp t;
    fp_sub(&t, &a->c0, &a->c1);
    fp_add(&r->c1, &a->c0, &a->c1);
    r->c0 = t;
}
static void fp2_norm(fp *n, const fp2 *a) { fp t; fp_sqr(n, &a->c0); fp_sqr(&t, &a->c1); fp_add(n, n, &t); }
static void fp2_inv(fp2 *r, const fp2 *a) {
    fp n, t;
    fp2_norm(&n, a);
    fp_inv(&n, &n);
    fp_mul(&r->c0, &a->c0, &n);
    fp_mul(&t, &a->c1, &n);
    fp_neg(&r->c1, &t);
}
static unsigned fp2_sgn0(const fp2 *a) {
    fp c0, c1;
    fp_from_mont(&c0, &a->c0);
    fp_from_mont(&c1, &a->c1);
    return (unsigned)((c0.l[0] & 1) | ((fp_is_zero(&c0) ? 1u : 0u) & (c1.l[0] & 1)));
}
/* sqrt given a root n of the norm (norm method, SURVEY Appendix A) */
static int fp2_sqrt_nr(fp2 *r, const fp2 *a, const fp *n) {
    fp d, t, x0, chk, inv, other;
    fp_add(&d, &a->c0, n);
    fp_mul(&d, &d, &C_INV2);
    if (fp_is_zero(&d)) { fp_sub(&d, &a->c0, n); fp_mul(&d, &d, &C_INV2); }
    fp_pow_pm3d4(&t, &d);
    fp_mul(&x0, &t, &d);
    fp_sqr(&chk, &x0);
    int qr = fp_eq(&chk, &d);
    fp_mul(&inv, &t, &C_INV2);
    if (!qr) fp_neg(&inv, &inv);
    fp_mul(&other, &a->c1, &inv);
    if (qr) { r->c0 = x0; r->c1 = other; } else { r->c0 = other; r->c1 = x0; }
    fp2 sq;
    fp2_sqr(&sq, r);
    return fp2_eq(&sq, a);
}
static int fp2_sqrt(fp2 *r, const fp2 *a) {
    fp n, root;
    fp2_norm(&n, a);
    if (!fp_sqrt(&root, &n)) return 0;
    return fp2_sqrt_nr(r, a, &root);
}

/* ------------------------------------------------------------------------------------------------ Fp6 / Fp12 */
static void fp6_add(fp6 *r, const fp6 *a, const fp6 *b) { fp2_add(&r->c0, &a->c0, &b->c0); fp2_add(&r->c1, &a->c1, &b->c1); fp2_add(&r->c2, &a->c2, &b->c2); }
static void fp6_sub(fp6 *r, const fp6 *a, const fp6 *b) { fp2_sub(&r->c0, &a->c0, &b->c0); fp2_sub(&r->c1, &a->c1, &b->c1); fp2_sub(&r->c2, &a->c2, &b->c2); }
static void fp6_neg(fp6 *r, const fp6 *a) { fp2_neg(&r->c0, &a->c0); fp2_neg(&r->c1, &a->c1); fp2_neg(&r->c2, &a->c2); }
static void fp6_mul_v(fp6 *r, const fp6 *a) {
    fp2 t;
    fp2_mul_xi(&t, &a->c2);
    r->c2 = a->c1; r->c1 = a->c0; r->c0 = t;
}
static void fp6_mul(fp6 *r, const fp6 *a, const fp6 *b) {
    fp2 v0, v1, v2, t0, t1, t2, c0, c1, c2;
    fp2_mul(&v0, &a->c0, &b->c0); fp2_mul(&v1, &a->c1, &b->c1); fp2_mul(&v2, &a->c2, &b->c2);
    fp2_add(&t0, &a->c1, &a->c2); fp2_add(&t1, &b->c1, &b->c2); fp2_mul(&t2, &t0, &t1);
    fp2_sub(&t2, &t2, &v1); fp2_sub(&t2, &t2, &v2); fp2_mul_xi(&t2, &t2); fp2_add(&c0, &t2, &v0);
    fp2_add(&t0, &a->c0, &a->c1); fp2_add(&t1, &b->c0, &b->c1); fp2_mul(&t2, &t0, &t1);
    fp2_sub(&t2, &t2, &v0); fp2_sub(&t2, &t2, &v1); fp2_mul_xi(&t0, &v2); fp2_add(&c1, &t2, &t0);
    fp2_add(&t0, &a->c0, &a->c2); fp2_add(&t1, &b->c0, &b->c2); fp2_mul(&t2, &t0, &t1);
    fp2_sub(&t2, &t2, &v0); fp2_sub(&t2, &t2, &v2); fp2_add(&c2, &t2, &v1);
    r->c0 = c0; r->c1 = c1; r->c2 = c2;
}
static void fp6_mul_by_01(fp6 *r, const fp6 *a, const fp2 *b0, const fp2 *b1) {
    fp2 v0, v1, t0, t1, t2, c0, c1, c2;
    fp2_mul(&v0, &a->c0, b0); fp2_mul(&v1, &a->c1, b1);
    fp2_mul(&t0, &a->c2, b1); fp2_mul_xi(&t0, &t0); fp2_add(&c0, &t0, &v0);
    fp2_add(&t0, &a->c0, &a->c1); fp2_add(&t1, b0, b1); fp2_mul(&t2, &t0, &t1);
    fp2_sub(&t2, &t2, &v0); fp2_sub(&c1, &t2, &v1);
    fp2_mul(&t0, &a->c2, b0); fp2_add(&c2, &t0, &v1);
    r->c0 = c0; r->c1 = c1; r->c2 = c2;
}
static void fp6_mul_by_1(fp6 *r, const fp6 *a, const fp2 *b1) {
    fp2 c0, c1, c2;
    fp2_mul(&c0, &a->c2, b1); fp2_mul_xi(&c0, &c0);
    fp2_mul(&c1, &a->c0, b1); fp2_mul(&c2, &a->c1, b1);
    r->c0 = c0; r->c1 = c1; r->c2 = c2;
}
static void fp6_inv(fp6 *r, const fp6 *a) {
    fp2 t0, t1, t2, d, s;
    fp2_sqr(&t0, &a->c0); fp2_mul(&s, &a->c1, &a->c2); fp2_mul_xi(&s, &s); fp2_sub(&t0, &t0, &s);
    fp2_sqr(&t1, &a->c2); fp2_mul_xi(&t1, &t1); fp2_mul(&s, &a->c0, &a->c1); fp2_sub(&t1, &t1, &s);
    fp2_sqr(&t2, &a->c1); fp2_mul(&s, &a->c0, &a->c2); fp2_sub(&t2, &t2, &s);
    fp2_mul(&d, &a->c2, &t1); fp2_mul(&s, &a->c1, &t2); fp2_add(&d, &d, &s); fp2_mul_xi(&d, &d);
    fp2_mul(&s, &a->c0, &t0); fp2_add(&d, &d, &s);
    fp2_inv(&d, &d);
    fp2_mul(&r->c0, &t0, &d); fp2_mul(&r->c1, &t1, &d); fp2_mul(&r->c2, &t2, &d);
}
static void fp12_one(fp12 *a) { memset(a, 0, sizeof *a); a->c0.c0.c0 = C_ONE; }
static int fp12_is_one(const fp12 *a) { fp12 o; fp12_one(&o); return memcmp(a, &o, sizeof o) == 0; }
static void fp12_conj(fp12 *r, const fp12 *a) { r->c0 = a->c0; fp6_neg(&r->c1, &a->c1); }
static void fp12_mul(fp12 *r, const fp12 *a, const fp12 *b) {
    fp6 t0, t1, s0, s1, m;
    fp6_mul(&t0, &a->c0, &b->c0); fp6_mul(&t1, &a->c1, &b->c1);
    fp6_add(&s0, &a->c0, &a->c1); fp6_add(&s1, &b->c0, &b->c1); fp6_mul(&m, &s0, &s1);
    fp6_sub(&m, &m, &t0); fp6_sub(&r->c1, &m, &t1);
    fp6_mul_v(&t1, &t1); fp6_add(&r->c0, &t0, &t1);
}
static void fp12_sqr(fp12 *r, const fp12 *a) {
    fp6 s, t, m, av;
    fp6_add(&s, &a->c0, &a->c1); fp6_mul_v(&av, &a->c1); fp6_add(&t, &a->c0, &av);
    fp6_mul(&m, &a->c0, &a->c1); fp6_mul(&s, &s, &t); fp6_sub(&s, &s, &m);
    fp6_mul_v(&t, &m); fp6_sub(&r->c0, &s, &t); fp6_add(&r->c1, &m, &m);
}
static void fp12_mul_by_014(fp12 *r, const fp12 *a, const fp2 *c0, const fp2 *c1, const fp2 *c4) {
    fp6 t0, t1, s;
    fp2 c14;
    fp6_mul_by_01(&t0, &a->c0, c0, c1); fp6_mul_by_1(&t1, &a->c1, c4);
    fp2_add(&c14, c1, c4); fp6_add(&s, &a->c0, &a->c1); fp6_mul_by_01(&s, &s, c0, &c14);
    fp6_sub(&s, &s, &t0); fp6_sub(&r->c1, &s, &t1);
    fp6_mul_v(&t1, &t1); fp6_add(&r->c0, &t0, &t1);
}
static void fp12_inv(fp12 *r, const fp12 *a) {
    fp6 t0, t1;
    fp6_mul(&t0, &a->c0, &a->c0); fp6_mul(&t1, &a->c1, &a->c1); fp6_mul_v(&t1, &t1); fp6_sub(&t0, &t0, &t1);
    fp6_inv(&t0, &t0);
    fp6_mul(&r->c0, &a->c0, &t0); fp6_mul(&t1, &a->c1, &t0); fp6_neg(&r->c1, &t1);
}
static void fp12_frob(fp12 *r, const fp12 *a) {
    fp2 t;
    fp2_conj(&r->c0.c0, &a->c0.c0);
    fp2_conj(&t, &a->c1.c0); fp2_mul(&r->c1.c0, &t, &C_FROB1[1]);
    fp2_conj(&t, &a->c0.c1); fp2_mul(&r->c0.c1, &t, &C_FROB1[2]);
    fp2_conj(&t, &a->c1.c1); fp2_mul(&r->c1.c1, &t, &C_FROB1[3]);
    fp2_conj(&t, &a->c0.c2); fp2_mul(&r->c0.c2, &t, &C_FROB1[4]);
    fp2_conj(&t, &a->c1.c2); fp2_mul(&r->c1.c2, &t, &C_FROB1[5]);
}
static void fp12_frob2(fp12 *r, const fp12 *a) {
    r->c0.c0 = a->c0.c0;
    fp2_mul_fp(&r->c1.c0, &a->c1.c0, &C_FROB2[1]); fp2_mul_fp(&r->c0.c1, &a->c0.c1, &C_FROB2[2]);
    fp2_mul_fp(&r->c1.c1, &a->c1.c1, &C_FROB2[3]); fp2_mul_fp(&r->c0.c2, &a->c0.c2, &C_FROB2[4]);
    fp2_mul_fp(&r->c1.c2, &a->c1.c2, &C_FROB2[5]);
}
static void fp4_sqr(fp2 *r0, fp2 *r1, const fp2 *a, const fp2 *b) {
    fp2 t0, t1, t2;
    fp2_sqr(&t0, a); fp2_sqr(&t1, b); fp2_add(&t2, a, b); fp2_sqr(&t2, &t2);
    fp2_sub(&t2, &t2, &t0); fp2_sub(r1, &t2, &t1); fp2_mul_xi(&t1, &t1); fp2_add(r0, &t0, &t1);
}
static void fp12_cyc_sqr(fp12 *r, const fp12 *a) { /* Granger-Scott */
    fp2 t0, t1, t2, t3, t4, t5, u, x5;
    fp12 o;
    fp4_sqr(&t0, &t1, &a->c0.c0, &a->c1.c1);
    fp4_sqr(&t2, &t3, &a->c1.c0, &a->c0.c2);
    fp4_sqr(&t4, &t5, &a->c0.c1, &a->c1.c2);
    fp2_sub(&u, &t0, &a->c0.c0); fp2_dbl(&u, &u); fp2_add(&o.c0.c0, &u, &t0);
    fp2_add(&u, &t1, &a->c1.c1); fp2_dbl(&u, &u); fp2_add(&o.c1.c1, &u, &t1);
    fp2_mul_xi(&x5, &t5);
    fp2_add(&u, &x5, &a->c1.c0); fp2_dbl(&u, &u); fp2_add(&o.c1.c0, &u, &x5);
    fp2_sub(&u, &t4, &a->c0.c2); fp2_dbl(&u, &u); fp2_add(&o.c0.c2, &u, &t4);
    fp2_sub(&u, &t2, &a->c0.c1); fp2_dbl(&u, &u); fp2_add(&o.c0.c1, &u, &t2);
    fp2_add(&u, &t3, &a->c1.c2); fp2_dbl(&u, &u); fp2_add(&o.c1.c2, &u, &t3);
    *r = o;
}

/* ------------------------------------------------------------------------------------------------ curves */
#define X_ABS 0xd201000000010000ull
typedef struct { fp X, Y, Z; } g1j;
typedef struct { fp x, y; int inf; } g1a;
typedef struct { fp2 X, Y, Z; } g2j;
typedef struct { fp2 x, y; int inf; } g2a;

#define DEF_CURVE(F, J, A, PFX)                                                                                     \
    static int PFX##_is_inf(const J *p) { return F##_is_zero(&p->Z); }                                              \
    static void PFX##_set_inf(J *p) { memset(p, 0, sizeof *p); }                                                     \
    static void PFX##_dbl(J *r, const J *p) {                                                                        \
        F A_, B_, C_, D_, E_, F_, t;                                                                                 \
        F##_sqr(&A_, &p->X); F##_sqr(&B_, &p->Y); F##_sqr(&C_, &B_);                                                 \
        F##_add(&t, &p->X, &B_); F##_sqr(&t, &t); F##_sub(&t, &t, &A_); F##_sub(&t, &t, &C_); F##_add(&D_, &t, &t);  \
        F##_add(&E_, &A_, &A_); F##_add(&E_, &E_, &A_); F##_sqr(&F_, &E_);                                           \
        F##_mul(&t, &p->Y, &p->Z); F##_add(&r->Z, &t, &t);                                                           \
        F##_sub(&F_, &F_, &D_); F##_sub(&r->X, &F_, &D_);                                                            \
        F##_sub(&t, &D_, &r->X); F##_mul(&t, &E_, &t);                                                               \
        F##_add(&C_, &C_, &C_); F##_add(&C_, &C_, &C_); F##_add(&C_, &C_, &C_); F##_sub(&r->Y, &t, &C_);             \
    }                                                                                                                \
    static void PFX##_add(J *r, const J *p, const J *q) {                                                            \
        if (PFX##_is_inf(q)) { *r = *p; return; }                                                                    \
        if (PFX##_is_inf(p)) { *r = *q; return; }                                                                    \
        F Z1Z1, Z2Z2, U1, U2, S1, S2, H, I, Jv, rr, V, t, Z3, X3;                                                    \
        F##_sqr(&Z1Z1, &p->Z); F##_sqr(&Z2Z2, &q->Z); F##_mul(&U1, &p->X, &Z2Z2); F##_mul(&U2, &q->X, &Z1Z1);        \
        F##_mul(&S1, &p->Y, &q->Z); F##_mul(&S1, &S1, &Z2Z2); F##_mul(&S2, &q->Y, &p->Z); F##_mul(&S2, &S2, &Z1Z1);  \
        F##_sub(&H, &U2, &U1); F##_sub(&rr, &S2, &S1);                                                               \
        if (F##_is_zero(&H)) { if (F##_is_zero(&rr)) PFX##_dbl(r, p); else PFX##_set_inf(r); return; }               \
        F##_add(&rr, &rr, &rr); F##_add(&I, &H, &H); F##_sqr(&I, &I); F##_mul(&Jv, &H, &I); F##_mul(&V, &U1, &I);    \
        F##_add(&t, &p->Z, &q->Z); F##_sqr(&t, &t); F##_sub(&t, &t, &Z1Z1); F##_sub(&t, &t, &Z2Z2);                  \
        F##_mul(&Z3, &t, &H);                                                                                        \
        F##_sqr(&t, &rr); F##_sub(&t, &t, &Jv); F##_sub(&t, &t, &V); F##_sub(&X3, &t, &V);                           \
        F##_sub(&t, &V, &X3); F##_mul(&t, &rr, &t); F##_mul(&S1, &S1, &Jv); F##_add(&S1, &S1, &S1);                  \
        F##_sub(&r->Y, &t, &S1); r->X = X3; r->Z = Z3;                                                               \
    }                                                                                                                \
    static void PFX##_from_affine(J *r, const A *a) {                                                                \
        if (a->inf) { PFX##_set_inf(r); return; }                                                                    \
        r->X = a->x; r->Y = a->y; memset(&r->Z, 0, sizeof r->Z); *(fp *)&r->Z = C_ONE;                               \
    }                                                                                                                \
    static void PFX##_add_affine(J *r, const J *p, const A *q) {                                                     \
        if (q->inf) { *r = *p; return; }                                                                             \
        if (PFX##_is_inf(p)) { PFX##_from_affine(r, q); return; }                                                    \
        F Z1Z1, U2, S2, H, HH, I, Jv, rr, V, t, Z3, X3;                                                              \
        F##_sqr(&Z1Z1, &p->Z); F##_mul(&U2, &q->x, &Z1Z1); F##_mul(&S2, &q->y, &p->Z); F##_mul(&S2, &S2, &Z1Z1);     \
        F##_sub(&H, &U2, &p->X); F##_sub(&rr, &S2, &p->Y);                                                           \
        if (F##_is_zero(&H)) {                                                                                       \
            if (F##_is_zero(&rr)) { J qq; PFX##_from_affine(&qq, q); PFX##_dbl(r, &qq); } else PFX##_set_inf(r);     \
            return;                                                                                                  \
        }                                                                                                            \
        F##_add(&rr, &rr, &rr); F##_sqr(&HH, &H); F##_add(&I, &HH, &HH); F##_add(&I, &I, &I);                        \
        F##_mul(&Jv, &H, &I); F##_mul(&V, &p->X, &I);                                                                \
        F##_add(&t, &p->Z, &H); F##_sqr(&t, &t); F##_sub(&t, &t, &Z1Z1); F##_sub(&Z3, &t, &HH);                      \
        F##_sqr(&t, &rr); F##_sub(&t, &t, &Jv); F##_sub(&t, &t, &V); F##_sub(&X3, &t, &V);                           \
        F##_sub(&t, &V, &X3); F##_mul(&t, &rr, &t); F##_mul(&Jv, &p->Y, &Jv); F##_add(&Jv, &Jv, &Jv);                \
        F##_sub(&r->Y, &t, &Jv); r->X = X3; r->Z = Z3;                                                               \
    }                                                                                                                \
    static void PFX##_neg(J *r, const J *p) { r->X = p->X; F##_neg(&r->Y, &p->Y); r->Z = p->Z; }                     \
    static void PFX##_to_affine(A *r, const J *p) {                                                                  \
        if (PFX##_is_inf(p)) { memset(r, 0, sizeof *r); r->inf = 1; return; }                                        \
        F zi, zi2;                                                                                                   \
        F##_inv(&zi, &p->Z); F##_sqr(&zi2, &zi); F##_mul(&r->x, &p->X, &zi2);                                        \
        F##_mul(&zi2, &zi2, &zi); F##_mul(&r->y, &p->Y, &zi2); r->inf = 0;                                           \
    }                                                                                                                \
    static void PFX##_mul_u64(J *r, const J *p, uint64_t k) {                                                        \
        J acc; PFX##_set_inf(&acc);                                                                                  \
        for (int i = 63; i >= 0; i--) { PFX##_dbl(&acc, &acc); if ((k >> i) & 1) PFX##_add(&acc, &acc, p); }         \
        *r = acc;                                                                                                    \
    }                                                                                                                \
    static void PFX##_mul_be32(J *r, const J *p, const uint8_t *k) {                                                 \
        J acc; PFX##_set_inf(&acc);                                                                                  \
        for (int i = 0; i < 256; i++) { PFX##_dbl(&acc, &acc); if ((k[i >> 3] >> (7 - (i & 7))) & 1) PFX##_add(&acc, &acc, p); } \
        *r = acc;                                                                                                    \
    }

DEF_CURVE(fp, g1j, g1a, g1)
DEF_CURVE(fp2, g2j, g2a, g2)

static void g2_psi(g2j *r, const g2j *p) {
    fp2 t;
    fp2_conj(&t, &p->X); fp2_mul(&r->X, &t, &C_PSI_CX);
    fp2_conj(&t, &p->Y); fp2_mul(&r->Y, &t, &C_PSI_CY);
    fp2_conj(&r->Z, &p->Z);
}
static void g2_psi2(g2j *r, const g2j *p) { fp2_mul_fp(&r->X, &p->X, &C_PSI2_CX); fp2_neg(&r->Y, &p->Y); r->Z = p->Z; }
static void g2_mul_x_abs(g2j *r, const g2j *p) {
    g2j acc = *p;
    for (int i = 62; i >= 0; i--) { g2_dbl(&acc, &acc); if ((X_ABS >> i) & 1) g2_add(&acc, &acc, p); }
    *r = acc;
}
static int g2_jac_eq(const g2j *a, const g2j *b) {
    int ia = g2_is_inf(a), ib = g2_is_inf(b);
    if (ia || ib) return ia && ib;
    fp2 za, zb, l, r;
    fp2_sqr(&za, &a->Z); fp2_sqr(&zb, &b->Z); fp2_mul(&l, &a->X, &zb); fp2_mul(&r, &b->X, &za);
    if (!fp2_eq(&l, &r)) return 0;
    fp2_mul(&za, &za, &a->Z); fp2_mul(&zb, &zb, &b->Z); fp2_mul(&l, &a->Y, &zb); fp2_mul(&r, &b->Y, &za);
    return fp2_eq(&l, &r);
}
static int g2_in_subgroup(const g2a *p) { /* psi(P) == [x]P */
    if (p->inf) return 1;
    g2j pj, xp, ps;
    g2_from_affine(&pj, p); g2_mul_x_abs(&xp, &pj); g2_neg(&xp, &xp); g2_psi(&ps, &pj);
    return g2_jac_eq(&ps, &xp);
}
static void g2_clear_cofactor(g2j *r, const g2j *p) { /* RFC 9380 App. G.3 */
    g2j t1, t2, t3, n;
    g2_mul_x_abs(&t1, p); g2_neg(&t1, &t1);
    g2_psi(&t2, p);
    g2_dbl(&t3, p); g2_psi2(&t3, &t3);
    g2_neg(&n, &t2); g2_add(&t3, &t3, &n);
    g2_add(&t2, &t1, &t2); g2_mul_x_abs(&t2, &t2); g2_neg(&t2, &t2);
    g2_add(&t3, &t3, &t2); g2_neg(&n, &t1); g2_add(&t3, &t3, &n);
    g2_neg(&n, p); g2_add(r, &t3, &n);
}

/* serialisation (ZCash format) */
static int g1_from_uncompressed(g1a *r, const uint8_t *b) { /* 0 ok, 1 inf, 2 bad */
    /* the 96-byte form: compression and sort flags clear, an infinity encoding all zero otherwise (blst's P1
     * deserialize; the library's keys are decoded by the same rules) */
    if (b[0] & 0xa0) return 2;
    if (b[0] & 0x40) {
        uint8_t nz = b[0] & 0x3f;
        for (int i = 1; i < 96; i++) nz |= b[i];
        if (nz) return 2;
        memset(r, 0, sizeof *r); r->inf = 1; return 1;
    }
    fp cx, cy;
    fp_from_be48(&cx, b); fp_from_be48(&cy, b + 48);
    cx.l[5] &= 0x1fffffffffffffffull;
    if (fp_canon_cmp(&cx, &C_P) >= 0 || fp_canon_cmp(&cy, &C_P) >= 0) return 2;
    fp_to_mont(&r->x, &cx); fp_to_mont(&r->y, &cy); r->inf = 0;
    return 0;
}
static void g1_to_uncompressed(uint8_t *b, const g1a *p) {
    if (p->inf) { memset(b, 0, 96); b[0] = 0x40; return; }
    fp c;
    fp_from_mont(&c, &p->x); fp_to_be48(b, &c);
    fp_from_mont(&c, &p->y); fp_to_be48(b + 48, &c);
}
static int fp2_lex_larger(const fp2 *y) {
    fp c0, c1;
    fp_from_mont(&c0, &y->c0); fp_from_mont(&c1, &y->c1);
    return fp_is_zero(&c1) ? fp_canon_cmp(&c0, &C_HALF) > 0 : fp_canon_cmp(&c1, &C_HALF) > 0;
}
static int g2_decompress(g2a *r, const uint8_t *b) { /* 0 ok, 1 inf, 2 bad */
    unsigned c = b[0] >> 7, inf = (b[0] >> 6) & 1, s = (b[0] >> 5) & 1;
    if (!c) return 2;
    fp c1, c0;
    fp_from_be48(&c1, b); fp_from_be48(&c0, b + 48);
    c1.l[5] &= 0x1fffffffffffffffull;
    if (inf) {
        if (!fp_is_zero(&c1) || !fp_is_zero(&c0) || s) return 2;
        memset(r, 0, sizeof *r); r->inf = 1;
        return 1;
    }
    if (fp_canon_cmp(&c1, &C_P) >= 0 || fp_canon_cmp(&c0, &C_P) >= 0) return 2;
    fp_to_mont(&r->x.c0, &c0); fp_to_mont(&r->x.c1, &c1);
    fp2 rhs, y;
    fp2_sqr(&rhs, &r->x); fp2_mul(&rhs, &rhs, &r->x); fp2_add(&rhs, &rhs, &C_G2B);
    if (!fp2_sqrt(&y, &rhs)) return 2;
    if ((unsigned)fp2_lex_larger(&y) != s) fp2_neg(&y, &y);
    r->y = y; r->inf = 0;
    return 0;
}
static void g2_compress(uint8_t *b, const g2a *p) {
    if (p->inf) { memset(b, 0, 96); b[0] = 0xc0; return; }
    fp c;
    fp_from_mont(&c, &p->x.c1); fp_to_be48(b, &c);
    fp_from_mont(&c, &p->x.c0); fp_to_be48(b + 48, &c);
    b[0] |= 0x80 | (fp2_lex_larger(&p->y) ? 0x20 : 0);
}

/* ------------------------------------------------------------------------------------------------ hash to G2 */
static const char DST[] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"; /* blst.rs:15 */
static void expand_xmd_256(const uint8_t *msg32, uint8_t *out) {
    uint8_t buf[160], b0[32], m[80];
    memset(buf, 0, 64); memcpy(buf + 64, msg32, 32);
    buf[96] = 1; buf[97] = 0; buf[98] = 0;
    memcpy(buf + 99, DST, 43); buf[142] = 43;
    orc_sha256(buf, 143, b0);
    memcpy(m + 33, DST, 43); m[76] = 43;
    memcpy(m, b0, 32); m[32] = 1;
    orc_sha256(m, 77, out);
    for (int k = 2; k <= 8; k++) {
        for (int i = 0; i < 32; i++) m[i] = b0[i] ^ out[32 * (k - 2) + i];
        m[32] = (uint8_t)k;
        orc_sha256(m, 77, out + 32 * (k - 1));
    }
}
static void fp_from_be64_mod(fp *r, const uint8_t *b) {
    fp hi, lo, t;
    memset(&hi, 0, sizeof hi); memset(&lo, 0, sizeof lo);
    for (int i = 0; i < 4; i++) {
        uint64_t vh = 0, vl = 0;
        for (int k = 0; k < 8; k++) { vh = (vh << 8) | b[8 * (3 - i) + k]; vl = (vl << 8) | b[32 + 8 * (3 - i) + k]; }
        hi.l[i] = vh; lo.l[i] = vl;
    }
    fp_mul(&t, &hi, &C_R2_256); fp_mul(&lo, &lo, &C_R2); fp_add(r, &t, &lo);
}
static void sswu(fp2 *x, fp2 *y, const fp2 *u) {
    fp2 tv1, tv2, x1n, x1d, xd2, D, N, t, a, one, target, y0, invD, y1, x1;
    fp2_sqr(&tv1, u); fp2_mul(&tv1, &tv1, &C_SSWU_Z);
    fp2_sqr(&tv2, &tv1); fp2_add(&tv2, &tv2, &tv1);
    memset(&one, 0, sizeof one); one.c0 = C_ONE;
    fp2_add(&x1n, &tv2, &one); fp2_mul(&x1n, &x1n, &C_SSWU_B);
    if (fp2_is_zero(&tv2)) x1d = C_SSWU_ZA;
    else { fp2_mul(&x1d, &tv2, &C_SSWU_A); fp2_neg(&x1d, &x1d); }
    fp2_sqr(&xd2, &x1d); fp2_mul(&D, &xd2, &x1d);
    fp2_sqr(&N, &x1n); fp2_mul(&t, &xd2, &C_SSWU_A); fp2_add(&N, &N, &t); fp2_mul(&N, &N, &x1n);
    fp2_mul(&t, &D, &C_SSWU_B); fp2_add(&N, &N, &t);
    fp2_mul(&a, &N, &D);
    fp na, t1, s, chk, inv_na, nN;
    fp2_norm(&na, &a); fp_pow_pm3d4(&t1, &na); fp_mul(&s, &na, &t1); fp_sqr(&chk, &s);
    int is_sq = fp_eq(&chk, &na);
    target = a;
    if (!is_sq) { fp2_mul(&target, &a, &C_SSWU_Z); fp_mul(&s, &s, &C_SQRT_M5); }
    fp2_sqrt_nr(&y0, &target, &s);
    fp_sqr(&inv_na, &t1); fp_sqr(&inv_na, &inv_na); fp_mul(&inv_na, &inv_na, &na);
    fp2_norm(&nN, &N); fp_mul(&inv_na, &inv_na, &nN);
    fp2_conj(&invD, &D); fp2_mul_fp(&invD, &invD, &inv_na);
    fp2_mul(&y1, &y0, &invD); fp2_mul(&x1, &x1n, &xd2); fp2_mul(&x1, &x1, &invD);
    if (is_sq) { *x = x1; *y = y1; }
    else { fp2_mul(x, &tv1, &x1); fp2_mul(y, &tv1, u); fp2_mul(y, y, &y1); }
    if (fp2_sgn0(u) != fp2_sgn0(y)) fp2_neg(y, y);
}
static void iso_map(g2j *r, const fp2 *x, const fp2 *y) {
    fp2 xn, xd, yn, yd, t, yd2, xd2;
    fp2_mul(&xn, &C_ISO_XNUM[3], x); fp2_add(&xn, &xn, &C_ISO_XNUM[2]);
    fp2_mul(&xn, &xn, x); fp2_add(&xn, &xn, &C_ISO_XNUM[1]);
    fp2_mul(&xn, &xn, x); fp2_add(&xn, &xn, &C_ISO_XNUM[0]);
    fp2_add(&xd, x, &C_ISO_XDEN[1]); fp2_mul(&xd, &xd, x); fp2_add(&xd, &xd, &C_ISO_XDEN[0]);
    fp2_mul(&yn, &C_ISO_YNUM[3], x); fp2_add(&yn, &yn, &C_ISO_YNUM[2]);
    fp2_mul(&yn, &yn, x); fp2_add(&yn, &yn, &C_ISO_YNUM[1]);
    fp2_mul(&yn, &yn, x); fp2_add(&yn, &yn, &C_ISO_YNUM[0]);
    fp2_add(&yd, x, &C_ISO_YDEN[2]); fp2_mul(&yd, &yd, x); fp2_add(&yd, &yd, &C_ISO_YDEN[1]);
    fp2_mul(&yd, &yd, x); fp2_add(&yd, &yd, &C_ISO_YDEN[0]);
    fp2_mul(&r->Z, &xd, &yd); fp2_sqr(&yd2, &yd); fp2_mul(&t, &xn, &xd); fp2_mul(&r->X, &t, &yd2);
    fp2_sqr(&xd2, &xd); fp2_mul(&t, &xd2, &xd); fp2_mul(&t, &t, &yd2); fp2_mul(&t, &t, &yn); fp2_mul(&r->Y, &t, y);
}
static void hash_to_g2(g2j *r, const uint8_t *msg32) {
    uint8_t uni[256];
    fp2 u0, u1, x, y;
    g2j q0, q1;
    expand_xmd_256(msg32, uni);
    fp_from_be64_mod(&u0.c0, uni); fp_from_be64_mod(&u0.c1, uni + 64);
    fp_from_be64_mod(&u1.c0, uni + 128); fp_from_be64_mod(&u1.c1, uni + 192);
    sswu(&x, &y, &u0); iso_map(&q0, &x, &y);
    sswu(&x, &y, &u1); iso_map(&q1, &x, &y);
    g2_add(&q0, &q0, &q1);
    g2_clear_cofactor(r, &q0);
}

/* ------------------------------------------------------------------------------------------------ pairing */
typedef struct { fp px, py, pz; } g1p3;
static void dbl_step(g2j *T, fp2 *c0, fp2 *c1, fp2 *c4, const g1p3 *P) {
    fp2 A, B, C, D, E, Fq, ZZ, t, Z3;
    fp2_sqr(&A, &T->X); fp2_sqr(&B, &T->Y); fp2_sqr(&ZZ, &T->Z); fp2_sqr(&C, &B);
    fp2_add(&t, &T->X, &B); fp2_sqr(&t, &t); fp2_sub(&t, &t, &A); fp2_sub(&t, &t, &C); fp2_add(&D, &t, &t);
    fp2_add(&E, &A, &A); fp2_add(&E, &E, &A); fp2_sqr(&Fq, &E);
    fp2_add(&t, &T->Y, &T->Z); fp2_sqr(&t, &t); fp2_sub(&t, &t, &B); fp2_sub(&Z3, &t, &ZZ);
    fp2_mul(c0, &E, &T->X); fp2_sub(c0, c0, &B); fp2_sub(c0, c0, &B);
    fp2_mul(c1, &E, &ZZ); fp2_neg(c1, c1);
    fp2_mul(c4, &Z3, &ZZ);
    fp2_mul_fp(c0, c0, &P->pz); fp2_mul_fp(c1, c1, &P->px); fp2_mul_fp(c4, c4, &P->py);
    fp2_sub(&Fq, &Fq, &D); fp2_sub(&T->X, &Fq, &D);
    fp2_sub(&t, &D, &T->X); fp2_mul(&t, &E, &t);
    fp2_add(&C, &C, &C); fp2_add(&C, &C, &C); fp2_add(&C, &C, &C);
    fp2_sub(&T->Y, &t, &C); T->Z = Z3;
}
static void add_step(g2j *T, fp2 *c0, fp2 *c1, fp2 *c4, const g2a *Q, const g1p3 *P) {
    fp2 Z1Z1, U2, S2, H, HH, I, J, rr, V, t, Z3, X3;
    fp2_sqr(&Z1Z1, &T->Z); fp2_mul(&U2, &Q->x, &Z1Z1); fp2_mul(&S2, &Q->y, &T->Z); fp2_mul(&S2, &S2, &Z1Z1);
    fp2_sub(&H, &U2, &T->X); fp2_sub(&rr, &S2, &T->Y); fp2_add(&rr, &rr, &rr);
    fp2_sqr(&HH, &H); fp2_add(&I, &HH, &HH); fp2_add(&I, &I, &I); fp2_mul(&J, &H, &I); fp2_mul(&V, &T->X, &I);
    fp2_add(&t, &T->Z, &H); fp2_sqr(&t, &t); fp2_sub(&t, &t, &Z1Z1); fp2_sub(&Z3, &t, &HH);
    fp2_sqr(&t, &rr); fp2_sub(&t, &t, &J); fp2_sub(&t, &t, &V); fp2_sub(&X3, &t, &V);
    fp2_sub(&t, &V, &X3); fp2_mul(&t, &rr, &t); fp2_mul(&J, &T->Y, &J); fp2_add(&J, &J, &J);
    fp2_sub(&T->Y, &t, &J); T->X = X3; T->Z = Z3;
    fp2_mul(c0, &rr, &Q->x); fp2_mul(&t, &Q->y, &Z3); fp2_sub(c0, c0, &t);
    fp2_neg(c1, &rr); *c4 = Z3;
    fp2_mul_fp(c0, c0, &P->pz); fp2_mul_fp(c1, c1, &P->px); fp2_mul_fp(c4, c4, &P->py);
}
static void miller_loop(fp12 *f, const g1p3 *P, const g2a *Q) {
    g2j T;
    g2_from_affine(&T, Q);
    fp2 c0, c1, c4;
    fp12_one(f);
    for (int i = 62; i >= 0; i--) {
        if (i != 62) fp12_sqr(f, f);
        dbl_step(&T, &c0, &c1, &c4, P);
        fp12_mul_by_014(f, f, &c0, &c1, &c4);
        if ((X_ABS >> i) & 1) { add_step(&T, &c0, &c1, &c4, Q, P); fp12_mul_by_014(f, f, &c0, &c1, &c4); }
    }
    fp12_conj(f, f);
}
static void cyc_pow_x(fp12 *r, const fp12 *a) { /* a^x, x < 0 */
    fp12 acc = *a;
    for (int i = 62; i >= 0; i--) { fp12_cyc_sqr(&acc, &acc); if ((X_ABS >> i) & 1) fp12_mul(&acc, &acc, a); }
    fp12_conj(r, &acc);
}
/* f^(3 (p^12-1)/r): same exponent as the device (3 is coprime to r) */
static void final_exp3(fp12 *r, const fp12 *fin) {
    fp12 f, t0, t1, t2;
    fp12_conj(&t0, fin); fp12_inv(&t1, fin); fp12_mul(&f, &t0, &t1);
    fp12_frob2(&t0, &f); fp12_mul(&f, &t0, &f);
    cyc_pow_x(&t0, &f); fp12_conj(&t1, &f); fp12_mul(&t0, &t0, &t1);
    cyc_pow_x(&t1, &t0); fp12_conj(&t2, &t0); fp12_mul(&t0, &t1, &t2);
    cyc_pow_x(&t1, &t0); fp12_frob(&t2, &t0); fp12_mul(&t0, &t1, &t2);
    cyc_pow_x(&t1, &t0); cyc_pow_x(&t1, &t1); fp12_frob2(&t2, &t0); fp12_mul(&t1, &t1, &t2);
    fp12_conj(&t2, &t0); fp12_mul(&t1, &t1, &t2);
    fp12_cyc_sqr(&t2, &f); fp12_mul(&t2, &t2, &f);
    fp12_mul(r, &t1, &t2);
}

/* ------------------------------------------------------------------------------------------------ batch verify */
struct vs_ctx {
    const uint8_t *sigs, *msgs, *pks;
    const uint32_t *offs;
    const uint64_t *rands;
    uint8_t *status;
    fp12 *fparts;   /* per-thread-range products */
    g2j *sparts;
    int *fail;
    uint64_t *muls;
    uint64_t n;
    int nparts;
};
static void vs_range(uint64_t lo, uint64_t hi, void *vctx) {
    struct vs_ctx *c = (struct vs_ctx *)vctx;
    /* which part am I?  ranges are n*i/t .. n*(i+1)/t */
    int part = 0;
    for (int i = 0; i < c->nparts; i++)
        if (c->n * (uint64_t)i / (uint64_t)c->nparts == lo) part = i;
    fp12 acc;
    fp12_one(&acc);
    g2j ssum;
    g2_set_inf(&ssum);
    g_mulcount = 0;
    for (uint64_t i = lo; i < hi; i++) {
        const uint8_t *sb = c->sigs + 96 * i;
        int allz = 1;
        for (int k = 0; k < 96; k++) if (sb[k]) { allz = 0; break; }
        uint8_t st = 0;
        g2a sig;
        if (allz) st = 1;
        else {
            int rc = g2_decompress(&sig, sb);
            if (rc == 2) st = 2;
            else if (!g2_in_subgroup(&sig)) st = 3;
        }
        uint32_t klo = c->offs[i], khi = c->offs[i + 1];
        g1j apk;
        g1_set_inf(&apk);
        if (!st && khi <= klo) st = 4;
        for (uint32_t j = klo; j < khi && !st; j++) {
            g1a a;
            if (g1_from_uncompressed(&a, c->pks + 96ull * j) == 2) { st = 6; break; }
            g1_add_affine(&apk, &apk, &a);
        }
        if (!st && g1_is_inf(&apk)) st = 5;
        if (st) { if (c->status) c->status[i] = st; *c->fail = 1; continue; }
        uint64_t r = c->rands[i];
        g1j rapk;
        g1_mul_u64(&rapk, &apk, r);
        g1p3 P;
        fp z2;
        fp_mul(&P.px, &rapk.X, &rapk.Z); P.py = rapk.Y; fp_sqr(&z2, &rapk.Z); fp_mul(&P.pz, &z2, &rapk.Z);
        g2j hj, sj, rs;
        g2a h;
        hash_to_g2(&hj, c->msgs + 32 * i);
        g2_to_affine(&h, &hj);
        fp12 f;
        miller_loop(&f, &P, &h);
        fp12_mul(&acc, &acc, &f);
        if (!sig.inf) { g2_from_affine(&sj, &sig); g2_mul_u64(&rs, &sj, r); g2_add(&ssum, &ssum, &rs); }
    }
    c->fparts[part] = acc;
    c->sparts[part] = ssum;
    c->muls[part] = g_mulcount;
}

/* bls::verify_signature_sets over the same SoA layout as the C ABI (include/lhb200.h).  Returns 1/0.
 * gt_out (optional, 576 bytes): final-exponentiated product (cube), canonical big-endian, tower order.
 * fp_muls (optional): total Fp multiplications performed (instrumented counter). */
EXPORT int orc_verify_signature_sets(const uint8_t *sigs, const uint8_t *msgs, const uint8_t *pks, const uint32_t *offs,
                                     const uint64_t *rands, uint32_t n, uint8_t *status, uint8_t *gt_out,
                                     uint64_t *fp_muls) {
    if (n == 0) return 0;
    int T = orc_num_threads();
    if (T < 1) T = 1;
    if ((uint64_t)T > n) T = (int)n;
    if (T > 256) T = 256;
    struct vs_ctx c;
    int fail = 0;
    c.sigs = sigs; c.msgs = msgs; c.pks = pks; c.offs = offs; c.rands = rands; c.status = status;
    c.fparts = (fp12 *)malloc(sizeof(fp12) * (size_t)T);
    c.sparts = (g2j *)malloc(sizeof(g2j) * (size_t)T);
    c.muls = (uint64_t *)calloc((size_t)T, 8);
    c.fail = &fail; c.n = n; c.nparts = T;
    if (status) memset(status, 0, n);
    /* orc_par_for splits into exactly min(threads, n/min_grain) ranges of the form n*i/t */
    orc_par_for(n, 1, vs_range, &c);
    int ok = 0;
    uint64_t muls = 0;
    g_mulcount = 0;
    if (!fail) {
        fp12 acc = c.fparts[0];
        g2j s = c.sparts[0];
        for (int i = 1; i < T; i++) { fp12_mul(&acc, &acc, &c.fparts[i]); g2_add(&s, &s, &c.sparts[i]); }
        if (!g2_is_inf(&s)) {
            g2a sa;
            g2_to_affine(&sa, &s);
            g1p3 P;
            P.px = C_G1X; fp_neg(&P.py, &C_G1Y); P.pz = C_ONE;
            fp12 f;
            miller_loop(&f, &P, &sa);
            fp12_mul(&acc, &acc, &f);
        }
        final_exp3(&acc, &acc);
        ok = fp12_is_one(&acc);
        if (gt_out) {
            const fp2 *cs[6] = {&acc.c0.c0, &acc.c0.c1, &acc.c0.c2, &acc.c1.c0, &acc.c1.c1, &acc.c1.c2};
            for (int k = 0; k < 6; k++) {
                fp t;
                fp_from_mont(&t, &cs[k]->c0); fp_to_be48(gt_out + 96 * k, &t);
                fp_from_mont(&t, &cs[k]->c1); fp_to_be48(gt_out + 96 * k + 48, &t);
            }
        }
    }
    for (int i = 0; i < T; i++) muls += c.muls[i];
    muls += g_mulcount;
    if (fp_muls) *fp_muls = muls;
    free(c.fparts); free(c.sparts); free(c.muls);
    return ok;
}

/* stage probes for the tests */
EXPORT void orc_hash_to_g2(const uint8_t *msg32, uint8_t *out96) {
    g2j j; g2a a;
    hash_to_g2(&j, msg32); g2_to_affine(&a, &j); g2_compress(out96, &a);
}
EXPORT int orc_sk_to_pk(const uint8_t *sk_be32, uint8_t *out96) {
    g1j g, r; g1a a;
    g.X = C_G1X; g.Y = C_G1Y; g.Z = C_ONE;
    g1_mul_be32(&r, &g, sk_be32); g1_to_affine(&a, &r); g1_to_uncompressed(out96, &a);
    return 0;
}
EXPORT void orc_sign(const uint8_t *sk_be32, const uint8_t *msg32, uint8_t *out96) {
    g2j h, r; g2a a;
    hash_to_g2(&h, msg32); g2_mul_be32(&r, &h, sk_be32); g2_to_affine(&a, &r); g2_compress(out96, &a);
}
