// tests/hostsim/group_sum_sim.cpp — TEST INFRASTRUCTURE: bls/group_sum.cuh (the per-message key sum of grouped
// batches) compiled for the host with the PTX carry chains emulated (LHB_HOSTSIM), so tests/test_hostsim_group_sum.py
// can run the segmented tree level by level against oracle/bls_ref.py without a GPU.  The test compiles it into a
// temporary directory; it is never linked into liblhb200.so.
#define LHB_HOSTSIM 1
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../lighthouse_b200/csrc/bls/fp.cuh"
#include "../../lighthouse_b200/csrc/bls/fp2.cuh"
#include "../../lighthouse_b200/csrc/bls/ec.cuh"
#include "../../lighthouse_b200/csrc/bls/pairing.cuh"
#include "../../lighthouse_b200/csrc/bls/group_sum.cuh"

using namespace lhb200::bls;
#define EXPORT extern "C" __attribute__((visibility("default")))

// k_g1_group_sum, every member position of every tree level in turn.  Set j's point is the uncompressed key p96[j],
// handed to the tree in the key stage's projective form of a Jacobian point with Z != 1; status[j] != 0 keeps set j
// out of its group's sum.  Group g owns members[offsets[g] .. offsets[g + 1]).  out96[g] = uncompressed sum of group g
// (zeros when skip[g] != 0).  Returns the number of tree levels run.
EXPORT int hs_group_sum(const uint8_t* p96, const uint8_t* status, const uint32_t* members, const uint32_t* offsets,
                        int n, int n_groups, uint8_t* out96, uint8_t* skip) {
    std::vector<G1Proj3> P(n), out(n_groups);
    std::vector<G1Jac> tmp(offsets[n_groups]);
    for (int j = 0; j < n; j++) {
        G1Affine a;
        if (g1_from_uncompressed(a, p96 + 96 * j) != DEC_OK) return -1;
        Fp s, s2, s3; fp_add(s, a.x, a.y); fp_sqr(s2, s); fp_mul(s3, s2, s);   // same point as (x s^2, y s^3, s)
        G1Jac jj; fp_mul(jj.X, a.x, s2); fp_mul(jj.Y, a.y, s3); jj.Z = s;
        g1proj3_from_jac(P[j], jj);
    }
    GroupSumArgs ga;
    ga.P = P.data(); ga.status = status; ga.pk_status = status; ga.members = members; ga.offsets = offsets;
    const uint32_t n_pos = offsets[n_groups];   // member positions (every set is a member on the device)
    ga.n = n_pos; ga.n_groups = (uint32_t)n_groups; ga.tmp = tmp.data(); ga.out_p = out.data(); ga.skip = skip;
    uint32_t max_group = 0;
    for (int g = 0; g < n_groups; g++) max_group = std::max(max_group, offsets[g + 1] - offsets[g]);
    uint64_t span = 1;
    int level = 0;
    do {
        for (uint32_t p = 0; p < n_pos; p++) group_sum_position(ga, (uint32_t)level, span, p);
        level++;
        span *= GROUP_CHUNK;
    } while (span < max_group);
    for (int g = 0; g < n_groups; g++) {
        memset(out96 + 96 * g, 0, 96);
        if (skip[g]) continue;
        Fp zi; fp_inv(zi, out[g].pz);
        G1Affine r; fp_mul(r.x, out[g].px, zi); fp_mul(r.y, out[g].py, zi); r.inf = 0;
        g1_to_uncompressed(out96 + 96 * g, r);
    }
    return level;
}
