// group_sum.cuh — per-message sums of the key-stage points, for batches whose sets share messages.
//
// prod_i e(r_i apk_i, H(m)) = e(sum_i r_i apk_i, H(m)) (bilinearity, apk_i in G1), so sets that sign the same message
// need one hash-to-G2 and one Miller loop between them.  The host groups the sets by message (bls_host.cu) into a CSR:
// members[offsets[g] .. offsets[g + 1]) are the sets of group g.  k_g1_group_sum adds r_i apk_i over the members whose
// two status codes are 0 and writes the sum in the Miller kernels' G1Proj3 form, with skip[g] != 0 when no member
// contributes or the sum is the point at infinity (the pair then contributes 1, like a failed set).
//
// Segmented tree: level l combines runs of GROUP_CHUNK values at stride GROUP_CHUNK^l inside each group, in place in
// `tmp` (indexed by member position), so every serial chain has at most GROUP_CHUNK additions and a group of m members
// takes ceil(log_GROUP_CHUNK m) levels (at least one).  A group is finished at the first level whose span covers it.
#pragma once
#include "pairing.cuh"

namespace lhb200 {
namespace bls {

constexpr uint32_t GROUP_CHUNK = 8;

// (A : B : C) with x = A / C, y = B / C (the key stage's (X Z, Y, Z^3))  ->  Jacobian (A C, B C^2, C)
LHB_HD LHB_INLINE void g1jac_from_proj3(G1Jac& r, const G1Proj3& p) {
    Fp c2;
    fp_sqr(c2, p.pz);
    fp_mul(r.X, p.px, p.pz);
    fp_mul(r.Y, p.py, c2);
    r.Z = p.pz;
}

struct GroupSumArgs {
    const G1Proj3* P;           // r_i apk_i of every set (key stage)
    const uint8_t* status;      // signature-stage codes
    const uint8_t* pk_status;   // key-stage codes
    const uint32_t* members;    // n set indices, grouped
    const uint32_t* offsets;    // n_groups + 1
    uint32_t n, n_groups;
    G1Jac* tmp;                 // n partial sums (by member position)
    G1Proj3* out_p;             // n_groups sums
    uint8_t* skip;              // n_groups flags
};

// The work of member position p at tree level `level` (span = GROUP_CHUNK^level).
LHB_HD LHB_INLINE void group_sum_position(const GroupSumArgs& a, uint32_t level, uint64_t span, uint32_t p) {
    uint32_t lo = 0, hi = a.n_groups;   // the group of p: offsets[lo] <= p < offsets[lo + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a.offsets[mid] <= p) lo = mid; else hi = mid;
    }
    const uint32_t start = a.offsets[lo], end = a.offsets[lo + 1], size = end - start;
    const uint64_t out_span = span * GROUP_CHUNK;
    if ((p - start) % out_span != 0) return;
    if (level > 0 && size <= span) return;   // finished at an earlier level
    G1Jac acc;
    jac_set_inf(acc);
    for (uint32_t j = 0; j < GROUP_CHUNK; j++) {
        const uint64_t q = p + j * span;
        if (q >= end) break;
        G1Jac x;
        if (level == 0) {
            const uint32_t i = a.members[q];
            if ((a.status[i] | a.pk_status[i]) != 0) continue;
            g1jac_from_proj3(x, a.P[i]);
        } else {
            x = a.tmp[q];
        }
        jac_add(acc, acc, x);
    }
    if (size > out_span) { a.tmp[p] = acc; return; }
    G1Proj3 r;
    const bool inf = jac_is_inf(acc);
    if (inf) { r.px = FP_ONE; r.py = FP_ONE; r.pz = FP_ONE; }
    else g1proj3_from_jac(r, acc);
    a.out_p[lo] = r;
    a.skip[lo] = inf ? 1 : 0;
}

#if !defined(LHB_HOSTSIM)
// One tree level over every member position (most positions return at once above level 0).
__global__ void __launch_bounds__(64) k_g1_group_sum(GroupSumArgs a, uint32_t level, uint64_t span) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.n) group_sum_position(a, level, span, p);
}

// Segmented passes (several batch checks in one launch): the sum of r_i sig_i over each segment of sets
// [seg_off[k], seg_off[k + 1]), the same tree as above on contiguous runs.  Level l combines runs of GROUP_CHUNK values at
// stride GROUP_CHUNK^l in place in `sig_r` (the signature kernels' r_i sig_i, infinity for a failed set); the level whose
// span covers segment k writes its sum to out[k].  Segments are not empty.
__global__ void __launch_bounds__(64) k_g2_segment_sum(G2Jac* __restrict__ sig_r, const uint32_t* __restrict__ seg_off,
                                                       uint32_t n, uint32_t n_seg, uint32_t level, uint64_t span,
                                                       G2Jac* __restrict__ out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    uint32_t lo = 0, hi = n_seg;   // the segment of p: seg_off[lo] <= p < seg_off[lo + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (seg_off[mid] <= p) lo = mid; else hi = mid;
    }
    const uint32_t start = seg_off[lo], end = seg_off[lo + 1], size = end - start;
    const uint64_t out_span = span * GROUP_CHUNK;
    if ((p - start) % out_span != 0) return;
    if (level > 0 && size <= span) return;   // finished at an earlier level
    G2Jac acc;
    jac_set_inf(acc);
    for (uint32_t j = 0; j < GROUP_CHUNK; j++) {
        const uint64_t q = p + j * span;
        if (q >= end) break;
        G2Jac x = sig_r[q];
        jac_add(acc, acc, x);
    }
    if (size > out_span) sig_r[p] = acc;
    else out[lo] = acc;
}
#endif

}  // namespace bls
}  // namespace lhb200
