// miller_coop.cuh — cooperative multi-pairing Miller loop with ALL state in shared memory (no local-memory stack).
//
// The pairing work behind blst's verify_multiple_aggregate_signatures (crypto/bls/src/impls/blst.rs:114-118):
// prod_i f_{|x|,Q_i}(P_i), conjugated (x < 0).  Round 1 ran one thread per group of sets with a 4.5 KB/thread stack
// that spilled 74 GB per 100 k-set launch to DRAM (VERDICT r1).  Here
//   * a GROUP of six lanes shares one Fp12 accumulator f = sum a_k w^k (Fp12 = Fp2[w]/(w^6 - xi)); lane t owns the Fp2
//     coefficient a_t.  f^2 and the sparse products f * l are SCHOOLBOOK in the w-basis: lane t computes its own
//     output coefficient as fused sums of products (sop.cuh: one reduction per sum, Karatsuba inside Fp2 on reduced
//     values only — no double-width glue; uniform code across the six lanes);
//   * every lane owns one SignatureSet per round: its point T (homogeneous projective, Costello-Lange-Naehrig doubling:
//     3 M + 6 S in Fp2), the line through it and the temporaries live in the lane's private shared-memory column —
//     18 Fp slots = 864 B per lane: 3 for the coefficient of f, 1 scratch, and SEVEN Fp2 slots whose roles (X, Y, Z of
//     T, four temporaries, the three line coefficients) are permuted after every step instead of copying results;
//   * a WARP is five independent groups (30 lanes; lanes 30-31 idle) and synchronises only with itself (__syncwarp):
//     eight warps are resident per SM and drift apart, so one warp's operand set-up / reductions / stores overlap the
//     others' multiply loops (a first version with block barriers and 24 slots had 6 warps per SM in lock step and
//     stalled on its barriers);
//   * every lane runs `rounds` sets; between rounds T is parked in global memory (L2), so the shared-memory footprint is
//     independent of the batch size and one squaring of f is shared by 6 * rounds sets.
// Line convention as in pairing.cuh:  l = c0 + c1 w^2 + c4 w^3 (scaled by Fp2 factors the final exponentiation kills):
//   doubling at T = (X, Y, Z):  c0 = (Y^2 - 3 b' Z^2) pz,  c1 = -3 X^2 px,  c4 = 2 Y Z py        (b' = 4 xi)
//   addition of Q to T:         c0 = (u X2 - v Y2) pz,  c1 = -u Z2 px,  c4 = v Z2 py,  u = Y2 Z1 - Y1 Z2, v = X2 Z1 - X1 Z2
// with the G1 argument given projectively as (px, py, pz) = (x_P pz, y_P pz, pz)  (pairing.cuh G1Proj3).
//
// The program is written once as a sequence of PHASES separated by warp barriers (MC_PHASE); the host build
// (tests/hostsim) runs the same phases lane by lane, so the whole cooperative algorithm is checked limb-exactly on the
// CPU against the oracle before it ever runs on a GPU.
#pragma once
#include "pairing.cuh"
#include "sop.cuh"

namespace lhb200 {
namespace bls {
namespace mc {

constexpr int S_F0 = 0, S_F1 = 1, S_FS = 2;      // own coefficient of f: (re, im, re + im)
constexpr int S_SCR = 3;
constexpr int S_W = 4;                            // seven Fp2 slots: S_W + 2 k
constexpr int NSLOT = 18;
constexpr int TWORDS = 6 * NL;                    // one projective G2 point

// roles of the seven Fp2 slots (uniform across the warp; permuted after every step)
struct Roles {
    int x, y, z;        // T
    int w0, w1, w2, w3; // free
    int l0, l1, l4;     // line coefficients (valid between a step and its sparse products; alias three of the others)
};
LHB_HD LHB_INLINE Roles roles_init() {
    Roles r;
    r.x = S_W; r.y = S_W + 2; r.z = S_W + 4; r.w0 = S_W + 6; r.w1 = S_W + 8; r.w2 = S_W + 10; r.w3 = S_W + 12;
    r.l0 = r.l1 = r.l4 = 0;
    return r;
}

template <int NT>
struct Geom {
    static constexpr int LANES_USED = (NT / 6) * 6;                              // whole groups of six
    static constexpr size_t REGION_WORDS = (size_t)NSLOT * NL * NT + NT / 4 + 8; // columns + active flags (bytes)
};
template <int NT>
constexpr size_t region_words() { return Geom<NT>::REGION_WORDS; }

// squaring schedule of lane t: four terms  a_i * a_j  (x = a_i times 2 and/or xi, y = a_j);  byte = i | j << 3 |
// dbl << 6 | xi << 7, 0xff = no term.  r_t = sum_{i+j = t} a_i a_j + xi sum_{i+j = t+6} a_i a_j.
#define LHB_SQT(i, j, d, x) ((uint8_t)((i) | ((j) << 3) | ((d) << 6) | ((x) << 7)))
LHB_CONST uint8_t SQR_TERMS[6][4] = {
    {LHB_SQT(0, 0, 0, 0), LHB_SQT(1, 5, 1, 1), LHB_SQT(2, 4, 1, 1), LHB_SQT(3, 3, 0, 1)},
    {LHB_SQT(0, 1, 1, 0), LHB_SQT(2, 5, 1, 1), LHB_SQT(3, 4, 1, 1), 0xff},
    {LHB_SQT(0, 2, 1, 0), LHB_SQT(1, 1, 0, 0), LHB_SQT(3, 5, 1, 1), LHB_SQT(4, 4, 0, 1)},
    {LHB_SQT(0, 3, 1, 0), LHB_SQT(1, 2, 1, 0), LHB_SQT(4, 5, 1, 1), 0xff},
    {LHB_SQT(0, 4, 1, 0), LHB_SQT(1, 3, 1, 0), LHB_SQT(2, 2, 0, 0), LHB_SQT(5, 5, 0, 1)},
    {LHB_SQT(0, 5, 1, 0), LHB_SQT(1, 4, 1, 0), LHB_SQT(2, 3, 1, 0), 0xff},
};

// NT = lanes of a warp region (32 on the device, any multiple of 6 on the host); the first NG * 6 lanes work.
template <int NT>
struct Lane {
    Col<NT> c;
    int lane, t;         // lane within the warp region; t = lane within its group of six
    bool idle;           // lanes beyond the last whole group (30, 31 on the device)
    uint8_t* act;        // active flags of the current round, one per lane of the warp
    bool active;         // this lane's set of the current round takes part
    bool extra;          // ... and it is the appended pair (-g1, sum r sig)
    uint32_t set;
    Fp ra, rb;           // result coefficient in flight between a compute phase and its store phase
};
template <int NT>
constexpr int lanes_used() { return Geom<NT>::LANES_USED; }

struct Args {
    const G1Proj3* P;
    const G2Jac* H;
    const uint8_t* status;     // signature stage
    const uint8_t* pk_status = nullptr;   // key stage; null: only `status` marks the sets to skip
    uint32_t n;                // sets in P / H / status / pk_status
    const G2Jac* extra_q;      // nullable: the pair (*extra_p, *extra_q) = (-g1, sum r sig) is appended as set n
    const G1Proj3* extra_p;
    uint32_t lo, hi;           // this warp's sets [lo, hi)
    uint32_t* scratch;         // this warp's parking area: rounds * 2 * TWORDS * NT words (T and Q per set)
};

template <int NT>
LHB_HD LHB_INLINE const G1Proj3* lane_p(const Lane<NT>& L, const Args& a) { return L.extra ? a.extra_p : a.P + L.set; }
// park / unpark one Fp2 slot (24 words at stride NT)
template <int NT>
LHB_HD LHB_INLINE void ld_fp2(const Col<NT>& c, int slot, const uint32_t* g) {
    uint32_t* q = c.base() + slot * NL * NT;
#pragma unroll 8
    for (int w = 0; w < 2 * NL; w++) q[w * NT] = g[w * NT];
}
template <int NT>
LHB_HD LHB_INLINE void st_fp2(uint32_t* g, const Col<NT>& c, int slot) {
    const uint32_t* q = c.base() + slot * NL * NT;
#pragma unroll 8
    for (int w = 0; w < 2 * NL; w++) g[w * NT] = q[w * NT];
}
template <int NT>
LHB_HD LHB_INLINE void park_point(uint32_t* g, const Col<NT>& c, const Roles& r) {
    st_fp2(g, c, r.x); st_fp2(g + 2 * NL * NT, c, r.y); st_fp2(g + 4 * NL * NT, c, r.z);
}
template <int NT>
LHB_HD LHB_INLINE void unpark_point(const Col<NT>& c, const Roles& r, const uint32_t* g) {
    ld_fp2(c, r.x, g); ld_fp2(c, r.y, g + 2 * NL * NT); ld_fp2(c, r.z, g + 4 * NL * NT);
}
// bind the lane to its set of round r
template <int NT>
LHB_HD LHB_INLINE void lane_select(Lane<NT>& L, const Args& a, uint32_t r) {
    const uint32_t n_total = a.n + (a.extra_q ? 1u : 0u);
    // sets are dealt to the GROUPS of the warp first (set j of a round -> group j mod NG, slot j / NG): a warp with few
    // sets keeps every group short, and the serial sparse products of a group are what an iteration waits for
    L.set = a.lo + r * Geom<NT>::LANES_USED + L.t * (Geom<NT>::LANES_USED / 6) + L.lane / 6;
    L.extra = false;
    bool act = L.set < a.hi && L.set < n_total;
    if (act) {
        if (L.set >= a.n) { L.extra = true; act = !jac_is_inf(*a.extra_q); }
        else act = (a.status[L.set] | (a.pk_status ? a.pk_status[L.set] : 0)) == 0 && !jac_is_inf(a.H[L.set]);
    }
    L.active = act;
    L.act[L.lane] = act ? 1 : 0;
}
template <int NT>
LHB_HD LHB_INLINE uint32_t* park_t(const Lane<NT>& L, const Args& a, uint32_t r) { return a.scratch + (size_t)(2 * r) * TWORDS * NT + L.lane; }
template <int NT>
LHB_HD LHB_INLINE uint32_t* park_q(const Lane<NT>& L, const Args& a, uint32_t r) { return a.scratch + (size_t)(2 * r + 1) * TWORDS * NT + L.lane; }

// ---- prologue of a round: Q = H(m) Jacobian (X, Y, Z) -> projective (X Z, Y, Z^3) = T; parked copy for the additions
template <int NT>
LHB_HD LHB_INLINE void phase_init_point(Lane<NT>& L, const Args& a, const Roles& r, uint32_t* q_park) {
    if (!L.active) return;
    const Col<NT>& c = L.c;
    const G2Jac& h = L.extra ? *a.extra_q : a.H[L.set];
    c.st2(r.w0, h.X); c.st2(r.y, h.Y); c.st2(r.w1, h.Z);
    c2_mul(c, r.x, r.w0, r.w1);
    c2_sqr(c, r.z, r.w1, S_SCR);
    c2_mul(c, r.z, r.z, r.w1);
    park_point(q_park, c, r);
}

// ---- doubling step: T <- 2T and its line.  54 multiply units (3 M + 6 S + 3 scalings); results land where their last
// operand died; roles_after_dbl gives the new roles (see the header).
template <int NT>
LHB_HD LHB_INLINE void phase_dbl(Lane<NT>& L, const Args& a, const Roles& r) {
    if (!L.active) return;
    const Col<NT>& c = L.c;
    const G1Proj3* P = lane_p(L, a);
    c2_sqr(c, r.w0, r.x, S_SCR); c2_triple(c, r.w0, r.w0); c2_neg(c, r.w0, r.w0);  // -3 X^2
    c2_mul_fp(c, r.w0, r.w0, &P->px);                                              // c1  -> w0
    c2_mul(c, r.w1, r.x, r.y); c2_half(c, r.w1, r.w1);                             // A = X Y / 2            (X dead)
    c2_add(c, r.x, r.y, r.z); c2_sqr(c, r.x, r.x, S_SCR);                          // (Y + Z)^2 -> x
    c2_sqr(c, r.w2, r.y, S_SCR);                                                   // B = Y^2 -> w2         (Y dead)
    c2_sqr(c, r.y, r.z, S_SCR);                                                    // C = Z^2 -> y          (Z dead)
    c2_sub(c, r.x, r.x, r.w2); c2_sub(c, r.x, r.x, r.y);                           // H = 2 Y Z -> x
    c2_mul_12xi(c, r.y, r.y);                                                      // E = 3 b' C -> y
    c2_sub(c, r.w3, r.w2, r.y); c2_mul_fp(c, r.w3, r.w3, &P->pz);                  // c0 = (B - E) pz -> w3
    c2_triple(c, r.z, r.y);                                                        // F = 3 E -> z
    c2_sub(c, r.z, r.w2, r.z);                                                     // B - F
    c2_mul(c, r.w1, r.w1, r.z);                                                    // X3 = A (B - F) -> w1
    c2_half(c, r.z, r.z); c2_sub(c, r.z, r.w2, r.z);                               // G = (B + F)/2 = B - (B - F)/2
    c2_sqr(c, r.z, r.z, S_SCR); c2_sqr(c, r.y, r.y, S_SCR); c2_triple(c, r.y, r.y);
    c2_sub(c, r.z, r.z, r.y);                                                      // Y3 = G^2 - 3 E^2 -> z  (E dead)
    c2_mul_fp(c, r.y, r.x, &P->py);                                                // c4 = H py -> y
    c2_mul(c, r.w2, r.w2, r.x);                                                    // Z3 = B H -> w2         (x free)
}
LHB_HD LHB_INLINE void roles_after_dbl(Roles& r) {
    Roles n;
    n.x = r.w1; n.y = r.z; n.z = r.w2;
    n.l0 = r.w3; n.l1 = r.w0; n.l4 = r.y;
    n.w0 = r.x; n.w1 = r.w3; n.w2 = r.w0; n.w3 = r.y;   // the line slots are free again after the sparse products
    r = n;
}

// ---- addition step: T <- T + Q (projective, add-1998-cmo-2) and the line through T and Q; seven slots suffice
template <int NT>
LHB_HD LHB_INLINE void phase_add(Lane<NT>& L, const Args& a, const Roles& r, const uint32_t* q_park) {
    if (!L.active) return;
    const Col<NT>& c = L.c;
    const G1Proj3* P = lane_p(L, a);
    const uint32_t *qx = q_park, *qy = q_park + 2 * NL * NT, *qz = q_park + 4 * NL * NT;   // X2, Y2, Z2
    const int A = r.x, B = r.y, C = r.z, D = r.w0, E = r.w1, F = r.w2, G = r.w3;
    c2_mul_g(c, D, qz, B);                                  // d = Y1 Z2
    c2_mul_g(c, E, qz, A);                                  // e = X1 Z2          (a, b free)
    c2_mul_g(c, F, qz, C);                                  // f = Z1 Z2
    c2_mul_g(c, A, qy, C); c2_sub(c, A, A, D);              // a = u = Y2 Z1 - Y1 Z2
    c2_mul_g(c, B, qx, C); c2_sub(c, B, B, E);              // b = v = X2 Z1 - X1 Z2   (c free)
    c2_sqr(c, C, B, S_SCR);                                 // c = vv
    c2_mul(c, G, B, C);                                     // g = vvv
    c2_mul(c, E, C, E);                                     // e = R = vv X1Z2
    c2_sqr(c, C, A, S_SCR);                                 // c = uu
    c2_mul(c, C, C, F);                                     // c = uu Z1Z2
    c2_sub(c, C, C, G); c2_sub(c, C, C, E); c2_sub(c, C, C, E);   // c = A = uu Z1Z2 - vvv - 2R
    c2_mul(c, F, G, F);                                     // f = Z3 = vvv Z1Z2
    c2_mul(c, D, G, D);                                     // d = vvv Y1Z2       (g free)
    c2_sub(c, E, E, C); c2_mul(c, E, A, E); c2_sub(c, E, E, D);   // e = Y3 = u (R - A) - vvv Y1Z2   (d free)
    c2_mul(c, D, B, C);                                     // d = X3 = v A       (c free)
    c2_mul_g(c, C, qx, A); c2_mul_g(c, G, qy, B); c2_sub(c, C, C, G);
    c2_mul_fp(c, C, C, &P->pz);                             // c = c0 = (u X2 - v Y2) pz
    c2_mul_g(c, G, qz, A); c2_neg(c, G, G); c2_mul_fp(c, G, G, &P->px);   // g = c1 = -u Z2 px   (a free)
    c2_mul_g(c, A, qz, B); c2_mul_fp(c, A, A, &P->py);      // a = c4 = v Z2 py   (b free)
}
LHB_HD LHB_INLINE void roles_after_add(Roles& r) {
    Roles n;
    n.x = r.w0; n.y = r.w1; n.z = r.w2;                     // X3 = d, Y3 = e, Z3 = f
    n.l0 = r.z; n.l1 = r.w3; n.l4 = r.x;                    // c, g, a
    n.w0 = r.y; n.w1 = r.z; n.w2 = r.w3; n.w3 = r.x;        // b, then the line slots
    r = n;
}

// The f-updates are sums of Fp2 products  sum_q u_q * a_q  computed Karatsuba-style WITHOUT double-width values:
//     S0 = sum u_q.0 a_q.0,   S1 = sum u_q.1 a_q.1,   S2 = sum (u_q.0 + u_q.1)(a_q.0 + a_q.1)      (three fused sums)
//     re = S0 - S1,   im = S2 - S0 - S1
// 3 K products + 3 reductions instead of the schoolbook 4 K + 2; the coefficient is stored as (re, im, re + im) so the
// y operand of the third sum streams from shared memory like the others.  S0 and S1 run as two interleaved windows,
// S2 as a single one (all three at once would need 3 K x-operands + 72 window registers).
template <int K, int NT>
LHB_HD LHB_INLINE void sum_fp2_products(Lane<NT>& L, const SopX<K>& x0, const SopX<K>& x1, const Col<NT>* ycol) {
    SopY<K> y0, y1, ys;
    y0.stride = NT; y1.stride = NT; ys.stride = NT;
#pragma unroll
    for (int q = 0; q < K; q++) { y0.base[q] = ycol[q].at(S_F0); y1.base[q] = ycol[q].at(S_F1); ys.base[q] = ycol[q].at(S_FS); }
    Fp s0, s1, s2;
    fp_sop2<K>(s0, s1, x0, y0, x1, y1);                      // X = Y = 1
    SopX<K> xs;
#pragma unroll
    for (int q = 0; q < K; q++) fp_add_nr(xs.x[q], x0.x[q], x1.x[q]);   // < 2p: X = 2, Y = 1, K X <= 8
    fp_sop1<K>(s2, xs, ys);
    fp_sub_inl(L.ra, s0, s1);
    fp_sub_inl(s2, s2, s0);
    fp_sub_inl(L.rb, s2, s1);
}
// ---- f <- f^2: lane t's coefficient (four Fp2 terms, schedule SQR_TERMS)
template <int NT>
LHB_HD LHB_INLINE void phase_sqr_compute(Lane<NT>& L) {
    const Col<NT> g = L.c.lane(-L.t);   // column of the group's lane 0
    SopX<4> x0, x1;
    Col<NT> yc[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint32_t e = SQR_TERMS[L.t][k];
        const bool valid = e != 0xff;
        const int i = valid ? (e & 7) : 0, j = valid ? ((e >> 3) & 7) : 0;
        Fp2 u;
        g.lane(i).ld2(u, S_F0);
        if (e & 0x40) { fp_add_inl(u.c0, u.c0, u.c0); fp_add_inl(u.c1, u.c1, u.c1); }
        if (e & 0x80) fp2_mul_xi_inl(u, u);
        if (!valid) { fp_set_zero(u.c0); fp_set_zero(u.c1); }
        x0.x[k] = u.c0; x1.x[k] = u.c1;
        yc[k] = g.lane(j);
    }
    sum_fp2_products<4>(L, x0, x1, yc);
}
// ---- f <- f * l(owner): lane t's coefficient  a_t c0 + xi^[t<2] a_{t-2} c1 + xi^[t<3] a_{t-3} c4
template <int NT>
LHB_HD LHB_INLINE void phase_sparse_compute(Lane<NT>& L, const Roles& r, int owner) {
    const Col<NT> g = L.c.lane(-L.t);
    if (!L.act[L.lane - L.t + owner]) return;   // uniform within the group
    const Col<NT> oc = g.lane(owner);
    Fp2 l0, l1, l4;
    oc.ld2(l0, r.l0); oc.ld2(l1, r.l1); oc.ld2(l4, r.l4);
    if (L.t < 2) fp2_mul_xi_inl(l1, l1);
    if (L.t < 3) fp2_mul_xi_inl(l4, l4);
    SopX<3> x0, x1;
    x0.x[0] = l0.c0; x0.x[1] = l1.c0; x0.x[2] = l4.c0;
    x1.x[0] = l0.c1; x1.x[1] = l1.c1; x1.x[2] = l4.c1;
    const int i1 = L.t >= 2 ? L.t - 2 : L.t + 4, i2 = L.t >= 3 ? L.t - 3 : L.t + 3;
    const Col<NT> yc[3] = {L.c, g.lane(i1), g.lane(i2)};
    sum_fp2_products<3>(L, x0, x1, yc);
}
// ---- f <- f * g (dense): lane t's coefficient  sum_i a_i b_{(t - i) mod 6} xi^[i > t]  of its OWN group's f times the f
// held by the six columns starting at `src0` (another group of this warp, or group 0 of another warp's region).
// Two fused sums of three Fp2 terms each (K X <= 8 forbids six at once).  Used by the product tree of the epilogue.
template <int NT>
LHB_HD LHB_INLINE void phase_mul_compute(Lane<NT>& L, const Col<NT>& src0) {
    const Col<NT> g = L.c.lane(-L.t);
    Fp acc_a, acc_b;
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
        SopX<3> x0, x1;
        Col<NT> yc[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int i = 3 * half + k;
            Fp2 u;
            g.lane(i).ld2(u, S_F0);
            if (i > L.t) fp2_mul_xi_inl(u, u);
            x0.x[k] = u.c0; x1.x[k] = u.c1;
            yc[k] = src0.lane(i > L.t ? L.t - i + 6 : L.t - i);
        }
        sum_fp2_products<3>(L, x0, x1, yc);
        if (half == 0) { acc_a = L.ra; acc_b = L.rb; }
    }
    fp_add_inl(L.ra, L.ra, acc_a);
    fp_add_inl(L.rb, L.rb, acc_b);
}

template <int NT>
LHB_HD LHB_INLINE void phase_store_f(Lane<NT>& L) {
    Fp s;
    fp_add_inl(s, L.ra, L.rb);
    L.c.st(S_F0, L.ra); L.c.st(S_F1, L.rb); L.c.st(S_FS, s);
}
template <int NT>
LHB_HD LHB_INLINE void phase_store_f_if(Lane<NT>& L, int owner) {
    if (L.act[L.lane - L.t + owner]) phase_store_f(L);
}

// The whole program of one warp: PHASES separated by warp barriers.  MC_PHASE(stmts) runs stmts on the lane `L` (idle
// lanes skip them) and synchronises the warp (device), or runs them on every lane of `ex.lanes` in turn (host).
#ifdef LHB_HOSTSIM
#define MC_PHASE(...) do { for (auto& L : ex.lanes) { if (!L.idle) { __VA_ARGS__; } } } while (0)
#else
#define MC_PHASE(...) do { Lane<NT>& L = ex.L; if (!L.idle) { __VA_ARGS__; } __syncwarp(); } while (0)
#endif
template <int NT, class Exec>
LHB_HD LHB_INLINE void miller_program(Exec& ex, const Args& a) {
    constexpr int LU = Geom<NT>::LANES_USED;
    const uint32_t cnt = a.hi - a.lo;
    const uint32_t rounds = (cnt + LU - 1) / LU;
    Roles R = roles_init();
    // f = 1; points
    MC_PHASE(Fp z; fp_set_zero(z); Fp one = FP_ONE;
             L.c.st(S_F0, L.t == 0 ? one : z); L.c.st(S_F1, z); L.c.st(S_FS, L.t == 0 ? one : z));
    for (uint32_t r = 0; r < rounds; r++)
        MC_PHASE(lane_select(L, a, r);
                 phase_init_point(L, a, R, park_q(L, a, r));
                 if (rounds > 1 && L.active) park_point(park_t(L, a, r), L.c, R));
#pragma unroll 1
    for (int it = 62; it >= 0; it--) {
        MC_PHASE(phase_sqr_compute(L));
        MC_PHASE(phase_store_f(L));
        const int steps = ((BLS_X_ABS >> it) & 1) ? 2 : 1;
        const Roles R_in = R;       // every round starts from the same roles (T is (un)parked by role, not by slot)
        Roles R_out = R;
#pragma unroll 1
        for (uint32_t r = 0; r < rounds; r++) {
            R = R_in;
#pragma unroll 1
            for (int step = 0; step < steps; step++) {
                if (step == 0) {
                    MC_PHASE(if (rounds > 1) { lane_select(L, a, r); if (L.active) unpark_point(L.c, R, park_t(L, a, r)); }
                             phase_dbl(L, a, R));
                    roles_after_dbl(R);
                    if (steps == 1 && rounds > 1) MC_PHASE(if (L.active) park_point(park_t(L, a, r), L.c, R));
                } else {
                    MC_PHASE(phase_add(L, a, R, park_q(L, a, r)));
                    roles_after_add(R);
                    if (rounds > 1) MC_PHASE(if (L.active) park_point(park_t(L, a, r), L.c, R));
                }
#pragma unroll 1
                for (int owner = 0; owner < 6; owner++) {
                    MC_PHASE(phase_sparse_compute(L, R, owner));
                    MC_PHASE(phase_store_f_if(L, owner));
                }
            }
            R_out = R;
        }
        R = R_out;
    }
    // conjugate (x < 0): negate the odd powers of w (in place, keeping the (re, im, re + im) form)
    MC_PHASE(if (L.t & 1) {
                 Fp2 v; L.c.ld2(v, S_F0);
                 fp_neg(v.c0, v.c0); fp_neg(v.c1, v.c1);
                 L.ra = v.c0; L.rb = v.c1;
                 phase_store_f(L);
             });
    // product tree over the warp's groups: after it group 0 holds the product of all of them
    constexpr int NG = LU / 6;
    for (int stride = 1; stride < NG; stride *= 2) {
        MC_PHASE(const int gi = L.lane / 6;
                 L.active = (gi % (2 * stride) == 0) && gi + stride < NG;
                 if (L.active) phase_mul_compute(L, L.c.lane(-L.t + 6 * stride)));
        MC_PHASE(if (L.active) phase_store_f(L));
    }
}

// write group 0's f (the warp's product) in tower layout
template <int NT>
LHB_HD LHB_INLINE void store_group0(const Lane<NT>& L, Fp12& o) {
    if (L.idle || L.lane >= 6) return;
    Fp2 v;
    L.c.ld2(v, S_F0);
    Fp2& dst = L.t == 0 ? o.c0.c0 : L.t == 1 ? o.c1.c0 : L.t == 2 ? o.c0.c1 : L.t == 3 ? o.c1.c1 : L.t == 4 ? o.c0.c2 : o.c1.c2;
    dst = v;
}

#ifndef LHB_HOSTSIM
template <int NT>
struct ExecDev {
    Lane<NT>& L;
};

constexpr int MC_WARPS = 8;                       // warps per block = per SM
constexpr int MC_GROUPS_PER_WARP = 5;
constexpr size_t mc_smem_bytes() { return Geom<32>::REGION_WORDS * 4 * MC_WARPS; }

// One warp = 30 working lanes = 5 groups; global warp w (= warp_in_block * gridDim.x + blockIdx.x) owns sets
// [w * sets_per_warp, (w + 1) * sets_per_warp) of the n (+1) pairs.  The epilogue multiplies the groups of a warp and then the warps of the block together (the same
// cooperative w-basis product), so the kernel emits ONE Miller value per block: out_f[blockIdx.x].  scratch: per warp
// sets_per_warp rounded up to whole rounds of 30, 2 * TWORDS words per lane and round.
__global__ void __launch_bounds__(32 * MC_WARPS, 1) k_miller_coop(const G1Proj3* __restrict__ P, const G2Jac* __restrict__ H,
                                                                   const uint8_t* __restrict__ status,
                                                                   const uint8_t* __restrict__ pk_status, uint32_t n,
                                                                   const G2Jac* __restrict__ extra_q,
                                                                   const G1Proj3* __restrict__ extra_p,
                                                                   uint32_t sets_per_warp, uint32_t* __restrict__ scratch,
                                                                   Fp12* __restrict__ out_f) {
    constexpr int NT = 32;
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gw = wib * gridDim.x + blockIdx.x;   // interleaved: a batch of few warps spreads over all SMs
    uint32_t* region = lhb_dyn_smem + (size_t)wib * Geom<NT>::REGION_WORDS;
    Lane<NT> L;
    L.lane = lane;
    L.t = lane % 6;
    L.idle = lane >= Geom<NT>::LANES_USED;
    L.c = Col<NT>::make(region, lane);
    L.act = reinterpret_cast<uint8_t*>(region + NSLOT * NL * NT);
    L.active = false; L.extra = false; L.set = 0;
    const uint32_t n_total = n + (extra_q ? 1u : 0u);
    Args a;
    a.P = P; a.H = H; a.status = status; a.pk_status = pk_status; a.n = n; a.extra_q = extra_q; a.extra_p = extra_p;
    a.lo = min(n_total, gw * sets_per_warp);
    a.hi = min(n_total, a.lo + sets_per_warp);
    const uint32_t rounds_cap = (sets_per_warp + Geom<NT>::LANES_USED - 1) / Geom<NT>::LANES_USED;
    a.scratch = scratch + (size_t)gw * rounds_cap * 2 * TWORDS * NT;
    ExecDev<NT> ex{L};
    if (a.lo < a.hi) {
        miller_program<NT>(ex, a);
    } else if (!L.idle) {                       // a warp without sets contributes f = 1 to the block's product
        Fp z; fp_set_zero(z); Fp one = FP_ONE;
        L.c.st(S_F0, L.t == 0 ? one : z); L.c.st(S_F1, z); L.c.st(S_FS, L.t == 0 ? one : z);
    }
    // product over the block's warps (their group 0), then ONE Miller value per block
    for (int stride = 1; stride < MC_WARPS; stride *= 2) {
        __syncthreads();
        const bool mine = !L.idle && lane < 6 && (wib % (2 * stride) == 0) && wib + stride < MC_WARPS;
        if (mine) phase_mul_compute(L, Col<NT>::make(region + (size_t)stride * Geom<NT>::REGION_WORDS, 0));
        __syncthreads();
        if (mine) phase_store_f(L);
    }
    __syncthreads();
    if (wib == 0) store_group0(L, out_f[blockIdx.x]);
}
#endif

}  // namespace mc
}  // namespace bls
}  // namespace lhb200
