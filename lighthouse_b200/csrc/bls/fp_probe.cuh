// fp_probe.cuh — one base-field operation on raw little-endian limbs: the body of the batched field probe
// (lhb200_debug_fp_batch, one device thread per case) and of its host build (tests/hostsim).  The same source runs on
// both sides, so a test can require device == host == big integers case by case; where only the device disagrees the
// fault is in code generation or carry handling, not in the limb algorithm.
//
// No conversions: every operand and result is the raw 12-limb word array the arithmetic sees (Montgomery form where the
// operation assumes it).  Case layout: `in` holds the operands back to back (FP_PROBE_IN_WORDS[op] words); `out` gets
// up to three 12-limb results r0 | r1 | r2 and a flag word at FP_PROBE_FLAG.
#pragma once
#include "fp2.cuh"
#include "sop.cuh"

namespace lhb200 {
namespace bls {

enum FpProbeOp : int32_t {
    FPB_ADD = 0,            // r0 = a + b mod p              (a, b < p)
    FPB_SUB = 1,            // r0 = a - b mod p
    FPB_NEG = 2,            // r0 = -a mod p
    FPB_MUL = 3,            // r0 = a b / R mod p            (fp_mul)
    FPB_SQR = 4,            // r0 = a a / R mod p            (fp_sqr as the pipeline builds it)
    FPB_TO_MONT = 5,        // r0 = a R mod p
    FPB_FROM_MONT = 6,      // r0 = a / R mod p
    FPB_INV = 7,            // r0 = R^2 / a mod p (the Montgomery inverse; 0 -> 0), Fermat chain
    FPB_INV_VARTIME = 8,    // the same by the binary extended Euclidean algorithm
    FPB_SQRT = 9,           // r0 = candidate root, flag = 1 iff r0^2 == a
    FPB_LT_P = 10,          // flag = a < p                  (any 384-bit a)
    FPB_GT_HALF = 11,       // flag = a > (p - 1) / 2        (any 384-bit a)
    FPB_MUL_SPLIT = 12,     // r0 = fp_redc_inl(fp_mulw_inl(a, b))   (a, b < 2^384, a b < p R)
    FPB_SQR_DEDICATED = 13, // r0 = fp_sqr_inl(a)                    (a a < p R)
    FPB_FP2_MUL = 14,       // r0 | r1 = a * b in Fp2 (a = a0 | a1, b = b0 | b1, Montgomery form)
    FPB_FP2_SQR = 15,
    FPB_FP2_INV = 16,
    FPB_FP2_SQRT = 17,      // flag = 1 iff a root exists
    FPB_FP2_SGN0 = 18,      // flag = sgn0(a)
    FPB_SOP = 32,           // FPB_SOP + K, K in {1, 2, 4, 6, 8}: in = xa[K] | ya[K] | xb[K] | yb[K];
                            // r0 | r1 = fp_sop2<K>, r2 = fp_sop1<K>(xa, ya); y streamed at a stride other than 1
};
constexpr int FP_PROBE_FLAG = 3 * NL;
constexpr int FP_PROBE_OUT_WORDS = 3 * NL + 1;
constexpr int FP_PROBE_SOP_KMAX = 8;
constexpr int FP_PROBE_Y_WORDS = 2 * FP_PROBE_SOP_KMAX * NL;   // ya and yb of one case

// operand words of a case; 0 for an unknown op (the host side of the C ABI checks the caller's layout with it)
#ifdef LHB_HOSTSIM
inline int fp_probe_in_words(int op) {
#else
__host__ __device__ inline int fp_probe_in_words(int op) {
#endif
    switch (op) {
        case FPB_NEG: case FPB_SQR: case FPB_TO_MONT: case FPB_FROM_MONT: case FPB_INV: case FPB_INV_VARTIME:
        case FPB_SQRT: case FPB_LT_P: case FPB_GT_HALF: case FPB_SQR_DEDICATED:
            return NL;
        case FPB_ADD: case FPB_SUB: case FPB_MUL: case FPB_MUL_SPLIT:
        case FPB_FP2_SQR: case FPB_FP2_INV: case FPB_FP2_SQRT: case FPB_FP2_SGN0:
            return 2 * NL;
        case FPB_FP2_MUL:
            return 4 * NL;
        case FPB_SOP + 1: case FPB_SOP + 2: case FPB_SOP + 4: case FPB_SOP + 6: case FPB_SOP + 8:
            return 4 * (op - FPB_SOP) * NL;
    }
    return 0;
}

LHB_HD LHB_INLINE void fpb_ld(Fp& r, const uint32_t* w) {
#pragma unroll
    for (int i = 0; i < NL; i++) r.v[i] = w[i];
}
LHB_HD LHB_INLINE void fpb_st(uint32_t* w, const Fp& a) {
#pragma unroll
    for (int i = 0; i < NL; i++) w[i] = a.v[i];
}

// y operands are copied to `ycol` with limb j of operand q at ycol[(q * NL + j) * ystride] (yb after ya), the way the
// pipeline streams them from a shared-memory column
template <int K>
LHB_HD LHB_INLINE void fp_probe_sop(const uint32_t* in, uint32_t* ycol, int ystride, uint32_t* out) {
    SopX<K> xa, xb;
    SopY<K> ya, yb;
    ya.stride = ystride; yb.stride = ystride;
    for (int q = 0; q < K; q++) {
        fpb_ld(xa.x[q], in + q * NL);
        fpb_ld(xb.x[q], in + (2 * K + q) * NL);
        for (int j = 0; j < NL; j++) {
            ycol[(q * NL + j) * ystride] = in[(K + q) * NL + j];
            ycol[((K + q) * NL + j) * ystride] = in[(3 * K + q) * NL + j];
        }
        ya.base[q] = ycol + q * NL * ystride;
        yb.base[q] = ycol + (K + q) * NL * ystride;
    }
    Fp ra, rb, r1;
    fp_sop2<K>(ra, rb, xa, ya, xb, yb);
    fp_sop1<K>(r1, xa, ya);
    fpb_st(out, ra); fpb_st(out + NL, rb); fpb_st(out + 2 * NL, r1);
}

// Runs `op` on one case.  out[0 .. FP_PROBE_OUT_WORDS) is written in full (unused words 0).  Returns false for an
// unknown op.
LHB_HD inline bool fp_probe(int op, const uint32_t* in, uint32_t* ycol, int ystride, uint32_t* out) {
    for (int i = 0; i < FP_PROBE_OUT_WORDS; i++) out[i] = 0;
    Fp a, b, r;
    fp_set_zero(r);
    uint32_t flag = 0;
    if (op < FPB_SOP) {
        fpb_ld(a, in);
        if (fp_probe_in_words(op) >= 2 * NL) fpb_ld(b, in + NL);
    }
    switch (op) {
        case FPB_ADD: fp_add(r, a, b); break;
        case FPB_SUB: fp_sub(r, a, b); break;
        case FPB_NEG: fp_neg(r, a); break;
        case FPB_MUL: fp_mul(r, a, b); break;
        case FPB_SQR: fp_sqr(r, a); break;
        case FPB_TO_MONT: fp_to_mont(r, a); break;
        case FPB_FROM_MONT: fp_from_mont(r, a); break;
        case FPB_INV: fp_inv(r, a); break;
        case FPB_INV_VARTIME: fp_inv_vartime(r, a); break;
        case FPB_SQRT: flag = fp_sqrt(r, a) ? 1u : 0u; break;
        case FPB_LT_P: flag = fp_canon_lt_p(a) ? 1u : 0u; break;
        case FPB_GT_HALF: flag = fp_canon_gt_half(a) ? 1u : 0u; break;
        case FPB_MUL_SPLIT: { uint32_t w[2 * NL]; fp_mulw_inl(w, a, b); fp_redc_inl(r, w); } break;
        case FPB_SQR_DEDICATED: fp_sqr_inl(r, a); break;
        case FPB_FP2_MUL: case FPB_FP2_SQR: case FPB_FP2_INV: case FPB_FP2_SQRT: case FPB_FP2_SGN0: {
            Fp2 x, y, o;
            x.c0 = a; x.c1 = b;
            if (op == FPB_FP2_MUL) { fpb_ld(y.c0, in + 2 * NL); fpb_ld(y.c1, in + 3 * NL); }
            fp2_set_zero(o);
            if (op == FPB_FP2_MUL) fp2_mul(o, x, y);
            else if (op == FPB_FP2_SQR) fp2_sqr(o, x);
            else if (op == FPB_FP2_INV) fp2_inv(o, x);
            else if (op == FPB_FP2_SQRT) flag = fp2_sqrt(o, x) ? 1u : 0u;
            else flag = (uint32_t)fp2_sgn0(x);
            fpb_st(out, o.c0); fpb_st(out + NL, o.c1);
            out[FP_PROBE_FLAG] = flag;
            return true;
        }
        case FPB_SOP + 1: fp_probe_sop<1>(in, ycol, ystride, out); return true;
        case FPB_SOP + 2: fp_probe_sop<2>(in, ycol, ystride, out); return true;
        case FPB_SOP + 4: fp_probe_sop<4>(in, ycol, ystride, out); return true;
        case FPB_SOP + 6: fp_probe_sop<6>(in, ycol, ystride, out); return true;
        case FPB_SOP + 8: fp_probe_sop<8>(in, ycol, ystride, out); return true;
        default: return false;
    }
    fpb_st(out, r);
    out[FP_PROBE_FLAG] = flag;
    return true;
}

}  // namespace bls
}  // namespace lhb200
