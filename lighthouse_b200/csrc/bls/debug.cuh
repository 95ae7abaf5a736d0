// debug.cuh — single-thread stage probes used by the GPU parity tests (same stages as tests/hostsim):
// lets `pytest -m gpu` compare every stage of the BLS pipeline with the oracle, not just the final boolean.
// k_debug_fp_batch runs one base-field operation per thread over many cases (bls/fp_probe.cuh).
#pragma once
#include "kernels.cuh"
#include "coop.cuh"
#include "fp_probe.cuh"

namespace lhb200 {
namespace bls {

__device__ inline void dbg_fp_in(Fp& r, const uint8_t* be48) { Fp c; fp_from_be48(c, be48); fp_to_mont(r, c); }
__device__ inline void dbg_fp_out(uint8_t* be48, const Fp& a) { Fp c; fp_from_mont(c, a); fp_to_be48(be48, c); }
__device__ inline void dbg_fp2_in(Fp2& r, const uint8_t* b) { dbg_fp_in(r.c0, b); dbg_fp_in(r.c1, b + 48); }
__device__ inline void dbg_fp2_out(uint8_t* b, const Fp2& a) { dbg_fp_out(b, a.c0); dbg_fp_out(b + 48, a.c1); }
__device__ inline void dbg_fp12_out(uint8_t* b, const Fp12& f) {
    const Fp2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
    for (int i = 0; i < 6; i++) dbg_fp2_out(b + 96 * i, *c[i]);
}

// op codes documented in include/lhb200.h (lhb200_debug_bls)
__global__ void k_debug_bls(int op, const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int32_t* __restrict__ rc) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    *rc = 0;
    switch (op) {
        case 0: {  // expand_message_xmd: 32 -> 256
            uint8_t m[32], o[256];
            for (int i = 0; i < 32; i++) m[i] = in[i];
            expand_message_xmd_256(m, o);
            for (int i = 0; i < 256; i++) out[i] = o[i];
        } break;
        case 1: {  // hash_to_g2: 32 -> 96 compressed
            uint8_t m[32], o[96];
            for (int i = 0; i < 32; i++) m[i] = in[i];
            G2Jac j; hash_to_g2_jac(j, m);
            G2Affine a; jac_to_affine(a, j); g2_compress(o, a);
            for (int i = 0; i < 96; i++) out[i] = o[i];
        } break;
        case 2: {  // sswu: u (96) -> x|y (192)
            uint8_t b[96], o[192];
            for (int i = 0; i < 96; i++) b[i] = in[i];
            Fp2 u, x, y; dbg_fp2_in(u, b); map_to_curve_sswu(x, y, u);
            dbg_fp2_out(o, x); dbg_fp2_out(o + 96, y);
            for (int i = 0; i < 192; i++) out[i] = o[i];
        } break;
        case 3: {  // g2 decompress -> rc (DecodeStatus), out[0] = in-subgroup, out[1..97) = recompressed
            uint8_t b[96], o[96];
            for (int i = 0; i < 96; i++) b[i] = in[i];
            G2Affine a; *rc = g2_decompress(a, b);
            if (*rc != DEC_BAD) { out[0] = g2_in_subgroup(a) ? 1 : 0; g2_compress(o, a); for (int i = 0; i < 96; i++) out[1 + i] = o[i]; }
        } break;
        case 4: {  // g2 mul: 96 compressed | 8-byte LE scalar -> 96
            uint8_t b[96], o[96];
            for (int i = 0; i < 96; i++) b[i] = in[i];
            uint32_t k[2] = {0, 0};
            for (int i = 0; i < 8; i++) k[i >> 2] |= (uint32_t)in[96 + i] << (8 * (i & 3));
            G2Affine a; *rc = g2_decompress(a, b);
            G2Jac j; jac_mul_affine(j, a, k, 64);
            G2Affine r; jac_to_affine(r, j); g2_compress(o, r);
            for (int i = 0; i < 96; i++) out[i] = o[i];
        } break;
        case 5: {  // fp2 op: in = opcode byte | a(96) | b(96): 0 mul 1 sqr 2 inv 3 sqrt(rc=ok) 4 sgn0(rc)
            uint8_t b[193], o[96];
            for (int i = 0; i < 193; i++) b[i] = in[i];
            Fp2 x, y, r; dbg_fp2_in(x, b + 1); dbg_fp2_in(y, b + 97); r = x;
            switch (b[0]) {
                case 0: fp2_mul(r, x, y); break;
                case 1: fp2_sqr(r, x); break;
                case 2: fp2_inv(r, x); break;
                case 3: *rc = fp2_sqrt(r, x) ? 1 : 0; break;
                case 4: *rc = (int32_t)fp2_sgn0(x); break;
            }
            dbg_fp2_out(o, r);
            for (int i = 0; i < 96; i++) out[i] = o[i];
        } break;
        case 6: {  // pairing with final exp: g1 uncompressed 96 | g2 compressed 96 -> 576 (cube of GT)
            uint8_t b[192], o[576];
            for (int i = 0; i < 192; i++) b[i] = in[i];
            G1Affine p; G2Affine q;
            if (g1_from_uncompressed(p, b) != DEC_OK || g2_decompress(q, b + 96) != DEC_OK) { *rc = -1; break; }
            G1Proj3 pp; g1proj3_from_affine(pp, p);
            Fp12 f; miller_loop(f, pp, q); final_exp(f, f);
            dbg_fp12_out(o, f);
            for (int i = 0; i < 576; i++) out[i] = o[i];
        } break;
        case 7: {  // g1 sum of n keys: in = n (1 byte) | n*96 -> 96 uncompressed
            const int n = in[0];
            G1Jac acc; jac_set_inf(acc);
            for (int t = 0; t < n; t++) {
                uint8_t b[96];
                for (int i = 0; i < 96; i++) b[i] = in[1 + 96 * t + i];
                G1Affine a; if (g1_from_uncompressed(a, b) == DEC_BAD) { *rc = -1; return; }
                jac_add_affine(acc, acc, a);
            }
            G1Affine r; jac_to_affine(r, acc);
            uint8_t o[96]; g1_to_uncompressed(o, r);
            for (int i = 0; i < 96; i++) out[i] = o[i];
        } break;
        case 8: {  // sswu trace: u (96) -> 16 x 96
            uint8_t b[96];
            for (int i = 0; i < 96; i++) b[i] = in[i];
            Fp2 u, x, y, tr[16]; dbg_fp2_in(u, b); map_to_curve_sswu(x, y, u, tr);
            for (int k = 0; k < 16; k++) { uint8_t o[96]; dbg_fp2_out(o, tr[k]); for (int i = 0; i < 96; i++) out[96 * k + i] = o[i]; }
        } break;
        default: *rc = -100;
    }
}

// Batched field probe (lhb200_debug_fp_batch): one thread per case over as many blocks as the cases need.  The y
// operands of the sum-of-products ops are streamed from this block's shared memory at a stride of FP_PROBE_BLOCK words,
// the column layout the pipeline kernels use.
constexpr int FP_PROBE_BLOCK = 32;
__global__ void __launch_bounds__(FP_PROBE_BLOCK) k_debug_fp_batch(int op, const uint32_t* __restrict__ in, uint32_t n,
                                                                   uint32_t* __restrict__ out) {
    __shared__ uint32_t ycol[FP_PROBE_Y_WORDS * FP_PROBE_BLOCK];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int w = fp_probe_in_words(op);
    fp_probe(op, in + (size_t)w * i, ycol + threadIdx.x, FP_PROBE_BLOCK, out + (size_t)FP_PROBE_OUT_WORDS * i);
}

}  // namespace bls
}  // namespace lhb200
