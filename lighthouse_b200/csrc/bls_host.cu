// bls_host.cu — host driver + C ABI of the batch BLS verification path.
//
// Mirrors bls::verify_signature_sets (crypto/bls/src/impls/blst.rs:37-119) at the batch level: the caller (the
// Rust shim in INTEGRATION.md, or lighthouse_b200/bls.py) flattens SignatureSets into SoA buffers
//   sigs  n x 96 B  compressed G2            (AggregateSignature::serialize, generic_aggregate_signature.rs:153-160)
//   msgs  n x 32 B  signing roots            (generic_signature_set.rs:70)
//   pks   K x 96 B  uncompressed affine G1   (validator_pubkey_cache.rs:195-199 format), CSR offsets n+1
// and gets back the batch verdict.  All arithmetic runs on the device; there is no CPU fallback.
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <errno.h>
#include <sys/random.h>
#include <vector>
#include "bls/debug.cuh"
#include <condition_variable>
#include <thread>
#include <deque>
#include <string>
#include "ctx.h"

namespace lhb200 {

using namespace bls;

static inline uint32_t cdiv(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }

constexpr uint32_t GW_WPB = 4;   // warps per block of the one-warp-per-point G2 kernels (bls/g2_warp.cuh)

// What the batch driver takes from the device and the environment.  bls_init fills it under the context mutex before
// ctx().ready is set; it is read-only afterwards, so concurrent callers read it without a lock.
struct Config {
    uint32_t n_sm;
    uint32_t miller_occ;   // resident blocks per SM of k_miller_multi
    // switches (INTEGRATION.md): latency-mode kernels, cooperative Miller loop, TMA key sums, grouping, key staging
    bool g2_warp, miller_warp, miller_coop, final_warp, pk_tma, group_messages, stage_pageable;
};
static Config g_cfg;

static bool env_switch(const char* name, bool dflt) {
    const char* e = getenv(name);
    return e ? atoi(e) != 0 : dflt;
}

template <class K>
static bool reserve_smem(K* kernel, size_t bytes) {   // dynamic shared memory above the 48 KB default
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
}

int32_t bls_init() {
    Config c;
    int v = 0;
    LHB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, ctx().device));
    c.n_sm = (uint32_t)v;
    LHB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_miller_multi, MILLER_BLOCK, 0));
    c.miller_occ = (uint32_t)std::max(v, 1);
    c.g2_warp = env_switch("LHB_G2_WARP", true);
    c.miller_warp = env_switch("LHB_MILLER_WARP", true);
    c.miller_coop = env_switch("LHB_MILLER_COOP", true);
    c.final_warp = env_switch("LHB_FINAL_WARP", true);
    c.pk_tma = env_switch("LHB_PK_TMA", false);
    c.group_messages = env_switch("LHB_GROUP_MESSAGES", true);
    c.stage_pageable = env_switch("LHB_STAGE_PAGEABLE", true);
    // working sets (+ a shared-memory copy of the phase tables of the warp kernels)
    const size_t gw_smem = gw::smem_bytes(GW_WPB);
    if (!reserve_smem(gw::k_sig_prepare_warp, gw_smem) || !reserve_smem(gw::k_hash_to_g2_warp, gw_smem) ||
        !reserve_smem(gw::k_g2_sum_warp, gw_smem)) {
        set_error("g2 warp kernels: cannot reserve %zu B of shared memory", gw_smem);
        return LHB200_ECUDA;
    }
    if (!reserve_smem(mc::k_miller_coop, mc::mc_smem_bytes())) {
        set_error("k_miller_coop: cannot reserve %zu B of shared memory", mc::mc_smem_bytes());
        return LHB200_ECUDA;
    }
    if (!reserve_smem(mw::k_miller_warp, mw::smem_bytes(mc::MC_WARPS)) ||
        !reserve_smem(mw::k_miller_warp_segments, mw::smem_bytes(mc::MC_WARPS))) {
        set_error("k_miller_warp: cannot reserve shared memory");
        return LHB200_ECUDA;
    }
    if (!reserve_smem(fe::k_final_warp, fe::smem_bytes()) || !reserve_smem(fe::k_final_segments, fe::smem_bytes())) {
        set_error("k_final_warp: cannot reserve shared memory");
        return LHB200_ECUDA;
    }
    g_cfg = c;
    return LHB200_OK;
}
void bls_shutdown();

}  // namespace lhb200

using namespace lhb200;

// Groups sets by their 32-byte message: an open-addressing hash table over the messages (O(n) expected).  A fingerprint
// of all 32 bytes picks the bucket, and its high half is kept in the slot so that only a matching fingerprint costs a
// look at the stored message; two messages are equal when all 32 bytes match.  Groups come in order of first
// occurrence, the members of a group in ascending order.  Scratch is sized once (reserve).
struct MsgGrouper {
    std::vector<uint64_t> slot;   // (fingerprint >> 32) << 32 | (group + 1); 0 = empty
    std::vector<uint64_t> seen;   // pre-pass bitset over the fingerprints
    std::vector<uint32_t> gid, first, cnt, members, offsets;
    std::vector<uint8_t> msgs;   // one copy of each distinct message

    static uint32_t table_size(uint32_t n) {
        uint32_t t = 16;
        while (t < 2 * (uint64_t)n) t <<= 1;
        return t;
    }
    static uint64_t seen_bits(uint32_t n) { return (uint64_t)table_size(n) * 8; }   // >= 16 bits per message
    void reserve(uint32_t cap) {
        slot.resize(table_size(cap));
        seen.resize(seen_bits(cap) / 64);
        gid.resize(cap); first.resize(cap); cnt.resize(cap); members.resize(cap); offsets.resize(cap + 1);
        msgs.resize((size_t)cap * 32);
    }
    static uint64_t fingerprint(const uint8_t* m) {
        uint64_t w[4], h = 0x243F6A8885A308D3ull;
        memcpy(w, m, 32);
        for (int k = 0; k < 4; k++) {
            h = (h ^ w[k]) * 0x9E3779B97F4A7C15ull;
            h ^= h >> 32;
        }
        return h;
    }
    // Cheaper mix for the pre-pass below (one multiply); equal messages still get equal values.
    static uint64_t quick_fingerprint(const uint8_t* m) {
        uint64_t w[4];
        memcpy(w, m, 32);
        const uint64_t x = w[0] ^ ((w[1] << 17) | (w[1] >> 47)) ^ ((w[2] << 31) | (w[2] >> 33)) ^ ((w[3] << 47) | (w[3] >> 17));
        return x * 0x9E3779B97F4A7C15ull;
    }
    // -> number of distinct messages.  The CSR (members, offsets[0 .. n_groups]) and `msgs` are filled, and max_group set
    // to the size of the largest group, when at least `min_repeats` sets repeat a message (min_repeats 0: always).
    uint32_t run(const uint8_t* m, uint32_t n, uint32_t min_repeats, uint32_t* max_group) {
        *max_group = 0;
        if (min_repeats > 0) {
            // Pre-pass: a repeated message always finds its fingerprint bit set, so fewer bits found set than
            // min_repeats rules grouping out without the table (the common all-distinct batch; at >= 16 bits per
            // message the expected number of chance hits is about n / 32).
            const uint64_t bits = seen_bits(n), bmask = bits - 1;
            std::fill(seen.begin(), seen.begin() + bits / 64, 0ull);
            uint32_t hits = 0;
            for (uint32_t i = 0; i < n; i++) {
                const uint64_t b = (quick_fingerprint(m + (size_t)32 * i) >> 32) & bmask, bit = 1ull << (b & 63);
                hits += (seen[b >> 6] & bit) != 0;
                seen[b >> 6] |= bit;
            }
            if (hits < min_repeats) return n;
        }
        const uint32_t ts = table_size(n), mask = ts - 1;
        std::fill(slot.begin(), slot.begin() + ts, 0ull);
        uint32_t ng = 0;
        for (uint32_t i = 0; i < n; i++) {
            const uint8_t* mi = m + (size_t)32 * i;
            const uint64_t fp = fingerprint(mi), tag = fp & 0xFFFFFFFF00000000ull;
            for (uint32_t h = (uint32_t)fp & mask;; h = (h + 1) & mask) {
                const uint64_t s = slot[h];
                if (s == 0) {   // new message: group ng
                    slot[h] = tag | (ng + 1);
                    first[ng] = i;
                    cnt[ng] = 0;
                    gid[i] = ng++;
                    break;
                }
                const uint32_t g = (uint32_t)s - 1;
                if ((s & 0xFFFFFFFF00000000ull) == tag && memcmp(m + (size_t)32 * first[g], mi, 32) == 0) {
                    gid[i] = g;
                    break;
                }
            }
            cnt[gid[i]]++;
        }
        if (n - ng < min_repeats) return ng;
        offsets[0] = 0;
        for (uint32_t g = 0; g < ng; g++) {
            offsets[g + 1] = offsets[g] + cnt[g];
            *max_group = std::max(*max_group, cnt[g]);
            memcpy(&msgs[(size_t)32 * g], m + (size_t)32 * first[g], 32);
            cnt[g] = offsets[g];   // from here: the next free member slot of group g
        }
        for (uint32_t i = 0; i < n; i++) members[cnt[gid[i]]++] = i;
        return ng;
    }
};

struct lhb200_pubkey_table {
    G1Mont* d_keys = nullptr;
    uint64_t capacity = 0, len = 0;
};

struct lhb200_bls_batch {
    // indexed mode: keys come from a device-resident table
    const lhb200_pubkey_table* table = nullptr;
    uint32_t* d_indices = nullptr;
    uint64_t cap_indices = 0;
    uint32_t cap_sets = 0;
    uint64_t cap_keys = 0;
    uint32_t n = 0;
    // inputs (owned copies, or caller's device buffers)
    uint8_t *d_sigs = nullptr, *d_msgs = nullptr, *d_pks = nullptr;
    uint32_t* d_offsets = nullptr;
    uint64_t* d_rands = nullptr;
    const uint8_t *in_sigs = nullptr, *in_msgs = nullptr, *in_pks = nullptr;
    const uint32_t* in_offsets = nullptr;
    const uint64_t* in_rands = nullptr;
    // intermediates
    G2Jac* d_sigr = nullptr;      // r_i * sig_i
    G2Jac* d_sig_tmp[2] = {nullptr, nullptr};
    G1Proj3* d_p = nullptr;       // r_i * apk_i (projective evaluation point)
    G2Jac* d_h = nullptr;         // H(m_i), Jacobian
    Fp12* d_f = nullptr;          // Miller loop values
    Fp12* d_f_tmp[2] = {nullptr, nullptr};
    Fp12* d_flast = nullptr;
    Fp12* d_gt = nullptr;
    uint8_t* d_status = nullptr;     // signature-stage codes (1-3), zeroed per verify
    uint8_t* d_pk_status = nullptr;  // key-stage codes (0, 4-6), written for every set by the key kernels
    uint32_t* d_fail = nullptr;
    uint8_t* d_ok = nullptr;
    uint8_t* h_res = nullptr;     // pinned: ok, status (at 64), pk_status (at 64 + cap_sets)
    cudaStream_t s_main = nullptr;   // the stream lhb200_verify_signature_sets drives this handle on (one per handle)
    cudaStream_t s2 = nullptr, s3 = nullptr;
    cudaEvent_t e_h2c = nullptr, e_sig = nullptr;
    cudaEvent_t e_fork = nullptr, e_join = nullptr;
    cudaEvent_t e_k0 = nullptr, e_k1 = nullptr;  // around the Miller kernel, for the roofline
    cudaEvent_t e_done = nullptr;                // cudaEventBlockingSync: the host wait of long steps
    uint64_t launches_last = 0;
    // cooperative Miller kernel (bls/miller_coop.cuh): parking area for T / Q between rounds, the -g1 argument
    uint32_t* d_mc_scratch = nullptr;
    size_t mc_scratch_words = 0;
    G1Proj3* d_neg_g1 = nullptr;
    const G2Jac* d_sig_sum = nullptr;
    // small / medium batches: slice sums of the key lists (k_pk_partial -> k_pk_combine), PK_SLICES per set
    G1Jac* d_pk_part = nullptr;
    uint8_t* d_pk_part_bad = nullptr;
    // streamed key upload (lhb200_bls_batch_upload_async): the key copy is cut into chunks of whole sets on its own
    // stream; k_pk_aggregate runs per chunk as it lands while the signature / hash-to-curve kernels already compute
    static constexpr int MAX_CHUNKS = 16;
    static constexpr int N_PK_STREAMS = 4;
    cudaStream_t s_pk[N_PK_STREAMS] = {};    // high priority: chunk c is copied AND aggregated on s_pk[c % 4]
    cudaEvent_t e_pk[N_PK_STREAMS] = {};
    cudaEvent_t e_small = nullptr, e_copy_free = nullptr;
    uint32_t chunk_lo[MAX_CHUNKS + 1] = {};  // set ranges
    uint64_t chunk_key[MAX_CHUNKS + 1] = {}; // key ranges
    const uint8_t* h_pks = nullptr;          // caller's host keys (valid until result)
    int n_chunks = 0;                        // 0: inputs already complete on the device
    std::vector<uint64_t> rbuf;              // scalars drawn by the library (must outlive the async copy)
    uint32_t plan[LHB200_PLAN_WORDS] = {};   // kernels the last verify_enqueue chose (lhb200_bls_batch_plan)
    // sets grouped by message (host uploads where a message repeats): hash-to-G2 and Miller run per group
    uint32_t n_groups = 0;                   // 0: not grouped
    uint32_t max_group = 0;                  // members of the largest group (depth of the group-sum tree)
    MsgGrouper grouper;                      // host scratch + the CSR the device copies read
    uint32_t* d_members = nullptr;           // n set indices, grouped
    uint32_t* d_goffsets = nullptr;          // n_groups + 1
    uint8_t* d_gmsgs = nullptr;              // n_groups x 32 B, the distinct messages
    G1Proj3* d_gp = nullptr;                 // per-group sum of r_i apk_i
    uint8_t* d_gskip = nullptr;              // per group: nothing to pair (no contributing member, or the sum is O)
    G1Jac* d_gtmp = nullptr;                 // partial sums of the group-sum tree
    // segmented pass (lhb200_bls_batch_set_segments): independent batch checks over contiguous runs of sets
    uint32_t n_seg = 0;                      // segments of the next upload + verify_enqueue; 0: one batch
    uint32_t n_seg_last = 0;                 // segments of the last verify_enqueue (segment_result, segment_gt)
    uint32_t max_seg = 0;                    // sets of the largest segment
    std::vector<uint32_t> seg_h;             // set offsets (n_seg + 1), then pair offsets (n_seg + 1): copied to d_seg_off
    std::vector<uint32_t> seg_members, seg_goffsets;   // grouping within segments (the CSR d_members / d_goffsets get)
    std::vector<uint8_t> seg_gmsgs;
    // allocated on the first set_segments, sized for the largest pass (pass_limit())
    uint32_t* d_seg_off = nullptr;           // set offsets, then pair offsets
    G2Jac* d_seg_sig = nullptr;              // per segment: sum of r_i sig_i
    Fp12* d_seg_f = nullptr;                 // Miller values: one per pair, then one per segment
    Fp12* d_seg_gt = nullptr;
    uint8_t* d_seg_ok = nullptr;
    uint8_t* h_seg_ok = nullptr;             // pinned
};

static void batch_free(lhb200_bls_batch* b) {
    if (!b) return;
    if (b->d_indices) cudaFree(b->d_indices);
    void* ptrs[] = {b->d_sigs, b->d_msgs, b->d_pks, b->d_offsets, b->d_rands, b->d_sigr, b->d_sig_tmp[0],
                    b->d_sig_tmp[1], b->d_p, b->d_h, b->d_f, b->d_f_tmp[0], b->d_f_tmp[1], b->d_flast, b->d_gt,
                    b->d_status, b->d_pk_status, b->d_fail, b->d_ok, b->d_mc_scratch, b->d_neg_g1, b->d_pk_part,
                    b->d_pk_part_bad, b->d_members, b->d_goffsets, b->d_gmsgs, b->d_gp, b->d_gskip, b->d_gtmp,
                    b->d_seg_off, b->d_seg_sig, b->d_seg_f, b->d_seg_gt, b->d_seg_ok};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (b->h_res) cudaFreeHost(b->h_res);
    if (b->h_seg_ok) cudaFreeHost(b->h_seg_ok);
    if (b->s_main) cudaStreamDestroy(b->s_main);
    if (b->s2) cudaStreamDestroy(b->s2);
    if (b->s3) cudaStreamDestroy(b->s3);
    if (b->e_h2c) cudaEventDestroy(b->e_h2c);
    if (b->e_sig) cudaEventDestroy(b->e_sig);
    if (b->e_fork) cudaEventDestroy(b->e_fork);
    if (b->e_join) cudaEventDestroy(b->e_join);
    if (b->e_k0) cudaEventDestroy(b->e_k0);
    if (b->e_k1) cudaEventDestroy(b->e_k1);
    if (b->e_done) cudaEventDestroy(b->e_done);
    for (cudaStream_t st : b->s_pk)
        if (st) cudaStreamDestroy(st);
    for (cudaEvent_t e : b->e_pk)
        if (e) cudaEventDestroy(e);
    if (b->e_small) cudaEventDestroy(b->e_small);
    if (b->e_copy_free) cudaEventDestroy(b->e_copy_free);
    delete b;
}

constexpr uint32_t REDUCE_CHUNK = 8;
// latency modes of the per-set stages (batches that do not fill the GPU): slice-parallel key sums, two threads per hash
constexpr uint32_t PK_SPLIT_MAX_SETS = 8192;
constexpr uint32_t HASH_PAIR_MAX_SETS = 4096;    // (at 10 000 sets the plain kernel was the faster one)
constexpr uint32_t FINAL_WARP_TAIL = 160;             // Miller block products k_final_warp takes directly (one per SM + slack)
constexpr uint32_t BLOCKING_WAIT_MIN_SETS = 16384;   // lhb200_bls_batch_result: blocking wait for steps of tens of ms

constexpr uint32_t CTAS_PER_SM = 12;          // cap of the grid-stride kernels: fewer threads keep their 1-4 KB stacks in L1/L2
constexpr uint32_t G2_SUM_WARP_CHUNK = 4;     // points per warp and level of k_g2_sum_warp
constexpr uint32_t MC_LANES = 30;             // working lanes per warp of k_miller_coop

// Levels of a tree that combines `chunk` values per level until at most `limit` remain; *rest = the values left.
static uint32_t tree_levels(uint32_t m, uint32_t chunk, uint32_t limit, uint32_t* rest = nullptr) {
    uint32_t levels = 0;
    for (; m > limit; levels++) m = cdiv(m, chunk);
    if (rest) *rest = m;
    return levels;
}

// Launches `levels` levels of a reduction tree over the m values at `cur`: launch(in, m, m_out, out) combines runs of
// `chunk` values into m_out = ceil(m / chunk), alternately into tmp[0] and tmp[1].  Returns the last level's output.
template <class T, class Launch>
static const T* reduce_tree(const T* cur, uint32_t m, uint32_t chunk, uint32_t levels, T* const tmp[2], Launch launch) {
    for (uint32_t l = 0; l < levels; l++, m = cdiv(m, chunk)) {
        launch(cur, m, cdiv(m, chunk), tmp[l & 1]);
        cur = tmp[l & 1];
    }
    return cur;
}

// Blocks of the one-thread-per-set kernels over m sets.  Resident CTAs per SM are capped (grid-stride kernels); above
// the cap every thread takes ceil(m / cap threads) sets, balanced across the grid.
static uint32_t lane_grid(const Config& c, uint32_t m) {
    const uint32_t cap = c.n_sm * CTAS_PER_SM;
    const uint32_t g = cdiv(m, BLS_BLOCK);
    return g > cap ? cdiv(m, (uint64_t)cdiv(m, cap * BLS_BLOCK) * BLS_BLOCK) : g;
}

// Every kernel and launch shape of one verify_enqueue.  w is what lhb200_bls_batch_plan reports; the launches read it.
struct Plan {
    uint32_t w[LHB200_PLAN_WORDS] = {};
    uint32_t ng = 0;               // pairs of the hash, Miller and final stages: the sets, or the groups of a grouped batch
    uint32_t hash_grid = 0;
    uint32_t miller_out = 0;       // Fp12 values the Miller kernel writes: the product tree's input
    size_t mc_scratch_words = 0;   // k_miller_coop's parking area for T / Q between rounds
};

// Sets plus segments of one segmented pass: every pair (and every segment's pair (-g1, sum r sig)) has a warp of its
// own in one wave of k_miller_warp_segments (8 warps per block, one block per SM).
static uint32_t pass_limit(const Config& c) { return c.n_sm * mc::MC_WARPS; }

// The selection policy: kernels and shapes from the sizes alone.  n_groups: 0 = not grouped; n_seg: 0 = one batch, else
// the segments of a segmented pass (max_seg sets in the largest).
static Plan choose(const Config& c, uint32_t n, uint32_t n_groups, uint32_t max_group, bool indexed, uint32_t n_chunks,
                   bool pks_aligned, uint32_t n_seg, uint32_t max_seg) {
    Plan p;
    uint32_t* w = p.w;
    const uint32_t ng = p.ng = n_groups ? n_groups : n;
    w[LHB200_PLAN_N_SETS] = n;
    w[LHB200_PLAN_N_SM] = c.n_sm;
    w[LHB200_PLAN_GROUPS] = n_groups;
    w[LHB200_PLAN_LANE_GRID] = lane_grid(c, n);
    w[LHB200_PLAN_LANE_SETS_PER_THREAD] = cdiv(n, (uint64_t)w[LHB200_PLAN_LANE_GRID] * BLS_BLOCK);
    // latency mode of the two G2 stages (bls/g2_warp.cuh): one warp per signature / message while the batch is small
    // enough for the warps of one wave (four per block, at most two blocks per SM); measured crossover with the
    // lane-per-set kernels: ~1 000 sets
    const bool g2_warp = c.g2_warp && n <= 6 * c.n_sm, hash_warp = c.g2_warp && ng <= 6 * c.n_sm;
    w[LHB200_PLAN_SIG] = g2_warp ? LHB200_K_SIG_PREPARE_WARP : LHB200_K_SIG_PREPARE;
    w[LHB200_PLAN_SUM_LEVELS] = tree_levels(n, g2_warp ? G2_SUM_WARP_CHUNK : REDUCE_CHUNK, 1);
    if (w[LHB200_PLAN_SUM_LEVELS]) w[LHB200_PLAN_SUM] = g2_warp ? LHB200_K_G2_SUM_WARP : LHB200_K_G2_REDUCE;
    w[LHB200_PLAN_LAST_MILLER] = !c.miller_coop;
    // latency mode of the plain hash: two threads per message (one SSWU map each)
    w[LHB200_PLAN_HASH] = hash_warp ? LHB200_K_HASH_TO_G2_WARP
                          : ng <= HASH_PAIR_MAX_SETS ? LHB200_K_HASH_TO_G2_PAIR : LHB200_K_HASH_TO_G2;
    p.hash_grid = hash_warp ? cdiv(ng, GW_WPB) : ng <= HASH_PAIR_MAX_SETS ? cdiv(2 * ng, BLS_BLOCK) : lane_grid(c, ng);
    // Explicit keys: slice-parallel sums for small and medium batches (a 512-key list is 64 + 8 additions deep instead
    // of 512), one thread per set above.  Key ingest through the TMA unit (bulk async copies into a shared-memory ring;
    // 16-byte aligned keys) is opt-in: on the H100 the plain kernel is faster at every size measured (100 000 sets x 128
    // keys: 111.8 against 119.5 ms per step; 40 000 sets: 49.0 against 53.3 ms).  The ring needs a shared-memory
    // carve-out, and an SM running blocks of the (shared-memory-free, full-L1) k_sig_prepare / k_hash_to_g2 cannot take
    // a block with a different carve-out until it drains; the kernel itself is bound by stack traffic, not by key loads.
    w[LHB200_PLAN_KEY] = indexed ? LHB200_K_PK_AGGREGATE_INDEXED
                         : c.pk_tma && pks_aligned ? LHB200_K_PK_AGGREGATE_TMA
                         : n <= PK_SPLIT_MAX_SETS ? LHB200_K_PK_PARTIAL_COMBINE : LHB200_K_PK_AGGREGATE;
    w[LHB200_PLAN_KEY_CHUNKS] = n_chunks;
    if (n_groups) {   // until one run of GROUP_CHUNK^levels covers the largest group
        w[LHB200_PLAN_GROUP_SUM] = LHB200_K_G1_GROUP_SUM;
        w[LHB200_PLAN_GROUP_SUM_LEVELS] = std::max<uint32_t>(1, tree_levels(max_group, GROUP_CHUNK, 1));
    }
    if (n_seg) {
        // Segmented pass: the per-set stages above, then per segment its own sum of r sig (a tree over its run of sets),
        // its own pair (-g1, sum) and its own tail.  Miller in latency mode only, one value per warp: no product may
        // combine two segments.  The callers keep ng + n_seg <= n + n_seg <= pass_limit(c).
        const uint32_t n_total = ng + n_seg, wpb = n_total <= 4 * COOP_TAIL ? 4 : mc::MC_WARPS;
        w[LHB200_PLAN_SEGMENTS] = n_seg;
        w[LHB200_PLAN_SUM] = LHB200_K_G2_SEGMENT_SUM;
        w[LHB200_PLAN_SUM_LEVELS] = std::max<uint32_t>(1, tree_levels(max_seg, GROUP_CHUNK, 1));
        w[LHB200_PLAN_LAST_MILLER] = 0;
        w[LHB200_PLAN_MILLER] = LHB200_K_MILLER_WARP;
        w[LHB200_PLAN_MILLER_WPB] = wpb;
        w[LHB200_PLAN_MILLER_SPW] = 1;
        w[LHB200_PLAN_MILLER_GRID] = cdiv(n_total, wpb);
        p.miller_out = n_total;
        w[LHB200_PLAN_FINAL] = LHB200_K_FINAL_SEGMENTS;
        return p;
    }
    // Miller loops over the ng pairs and, except with k_miller_multi, the pair (-g1, sum r sig)
    const uint32_t n_total = ng + 1, max_warps = c.n_sm * mc::MC_WARPS;
    uint32_t tail_max = COOP_TAIL;   // Miller products the final kernel folds itself
    if (c.miller_coop && c.miller_warp && n_total <= max_warps) {
        // Latency mode (bls/miller_warp.cuh): while every pair can have a warp of its own in one wave, a whole warp runs
        // one Miller loop at Fp granularity, far shorter than a lane-per-set loop.  Four warps per block (one per
        // scheduler) up to 256 pairs, eight above; <= 64 block products need no k_fp12_reduce level.
        const uint32_t wpb = n_total <= 4 * COOP_TAIL ? 4 : mc::MC_WARPS;
        w[LHB200_PLAN_MILLER] = LHB200_K_MILLER_WARP;
        w[LHB200_PLAN_MILLER_WPB] = wpb;
        w[LHB200_PLAN_MILLER_SPW] = 1;
        w[LHB200_PLAN_MILLER_GRID] = p.miller_out = cdiv(n_total, wpb);
    } else if (c.miller_coop) {
        // Cooperative shared-memory Miller loop (bls/miller_coop.cuh): one block of 8 independent warps per SM, 30
        // working lanes per warp, every lane runs `rounds` sets, six lanes share one accumulator.  Small batches spread
        // over more, emptier warps (latency), large ones fill 8 x n_sm.
        uint32_t spw = cdiv(cdiv(n_total, max_warps), MC_LANES) * MC_LANES;   // sets per warp, whole rounds
        uint32_t n_warps, mgrid;
        // Batches below one full round per warp.  A warp's five groups take one set each at no extra latency (SIMT), and
        // every further set of a group adds one serial sparse product per iteration (81 multiply units for a 1-set
        // group, 141 for a full one).  Small batches therefore use at least five sets per warp, at most 256 warps, four
        // per block (one per scheduler): <= 64 block products, which the final kernel folds itself (no k_fp12_reduce
        // level, a level of single-thread latency).  Above that: as few sets per warp as the 8 x n_sm warp budget allows.
        constexpr uint32_t FEW_WARPS = 4 * COOP_TAIL;
        const bool few = n_total <= FEW_WARPS * MC_LANES;
        if (few) {
            spw = std::min<uint32_t>(MC_LANES, std::max<uint32_t>(5, cdiv(cdiv(n_total, FEW_WARPS), 5) * 5));
            n_warps = cdiv(n_total, spw);
            mgrid = cdiv(n_warps, 4);
        } else {
            if (n_total <= max_warps * MC_LANES) spw = std::max<uint32_t>(1, cdiv(n_total, max_warps));
            n_warps = cdiv(n_total, spw);
            // warps are dealt round-robin to blocks (gw = warp_in_block * grid + block): few warps spread over all SMs
            mgrid = std::max<uint32_t>(std::min<uint32_t>(c.n_sm, n_warps), cdiv(n_warps, mc::MC_WARPS));
        }
        const uint32_t rounds_cap = cdiv(spw, MC_LANES);
        w[LHB200_PLAN_MILLER] = LHB200_K_MILLER_COOP;
        w[LHB200_PLAN_MILLER_WPB] = mc::MC_WARPS;
        w[LHB200_PLAN_MILLER_SPW] = spw;
        w[LHB200_PLAN_MILLER_GRID] = p.miller_out = mgrid;   // one product per block
        w[LHB200_PLAN_MILLER_ROUNDS_CAP] = rounds_cap;
        w[LHB200_PLAN_MILLER_FEW_WARPS] = few;
        p.mc_scratch_words = (size_t)mgrid * mc::MC_WARPS * rounds_cap * 2 * mc::TWORDS * 32;
        // k_final_warp folds the block products itself (8 warps share the products): no single-thread product level
        if (c.final_warp) tail_max = FINAL_WARP_TAIL;
    } else {
        // Sets per thread: k = ceil(ng / resident threads) (<= MILLER_KMAX) share their Fp12 squarings in one thread, so
        // a 100 k batch is ONE wave of 3-set groups instead of three waves of single Miller loops.
        const uint32_t resident = c.n_sm * c.miller_occ * MILLER_BLOCK;
        const uint32_t mk = std::min<uint32_t>(cdiv(ng, resident), MILLER_KMAX);
        p.miller_out = cdiv(ng, mk);
        w[LHB200_PLAN_MILLER] = LHB200_K_MILLER_MULTI;
        w[LHB200_PLAN_MILLER_SPW] = mk;
        w[LHB200_PLAN_MILLER_GRID] = std::min<uint32_t>(cdiv(p.miller_out, MILLER_BLOCK), c.n_sm * c.miller_occ);
    }
    w[LHB200_PLAN_FP12_REDUCE_LEVELS] = tree_levels(p.miller_out, REDUCE_CHUNK, tail_max, &w[LHB200_PLAN_N_TAIL]);
    // k_final_warp takes no k_last_miller value: only the kernels that pair (-g1, sum r sig) themselves feed it
    w[LHB200_PLAN_FINAL] = c.final_warp && c.miller_coop ? LHB200_K_FINAL_WARP : LHB200_K_FINAL_COOP;
    return p;
}

// ---- pool of batch handles behind lhb200_verify_signature_sets -------------------------------------------------
namespace {
// ---------------------------------------------------------------------------------------------------------
// Pageable key buffers (what a Rust Vec is).  cudaMemcpyAsync from pageable memory is staged by the driver through its
// own bounce buffer on the calling thread, well below the rate of a copy from pinned memory.  For big pageable key buffers the library stages them itself: a ring of pinned blocks filled by
// a few copy threads (memcpy scales with threads, the DMA engine reads pinned memory at link speed) and drained by
// cudaMemcpyAsync on the chunk's stream, so the CPU copy of block i + 1 overlaps the DMA of block i.
constexpr size_t STAGE_BLOCK = 16u << 20;
constexpr int STAGE_SLOTS = 4, STAGE_THREADS = 4;
constexpr uint64_t STAGE_MIN_BYTES = 64ull << 20;   // below this the driver's own staging is as good
struct KeyStager {
    uint8_t* slot[STAGE_SLOTS] = {};
    cudaEvent_t free_ev[STAGE_SLOTS] = {};
    bool used[STAGE_SLOTS] = {};
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    const uint8_t* src = nullptr;
    uint8_t* dst = nullptr;
    size_t bytes = 0;
    uint64_t generation = 0;
    int pending = 0;
    bool quit = false, ok = false;
    uint64_t next = 0;

    bool init() {
        if (ok) return true;
        for (int i = 0; i < STAGE_SLOTS; i++) {
            if (cudaHostAlloc(reinterpret_cast<void**>(&slot[i]), STAGE_BLOCK, cudaHostAllocDefault) != cudaSuccess ||
                cudaEventCreateWithFlags(&free_ev[i], cudaEventDisableTiming | cudaEventBlockingSync) != cudaSuccess) {
                cudaGetLastError();
                return false;
            }
        }
        for (int t = 0; t < STAGE_THREADS; t++) workers.emplace_back([this, t] { run(t); });
        ok = true;
        return true;
    }
    void run(int t) {
        uint64_t seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> lk(mu);
            cv_work.wait(lk, [&] { return quit || generation != seen; });
            if (quit) return;
            seen = generation;
            const uint8_t* s_ = src; uint8_t* d_ = dst; const size_t n = bytes;
            lk.unlock();
            const size_t per = (n + STAGE_THREADS - 1) / STAGE_THREADS, lo = std::min(n, per * t), hi = std::min(n, lo + per);
            if (hi > lo) memcpy(d_ + lo, s_ + lo, hi - lo);
            lk.lock();
            if (--pending == 0) cv_done.notify_one();
        }
    }
    void parallel_copy(uint8_t* d_, const uint8_t* s_, size_t n) {
        std::unique_lock<std::mutex> lk(mu);
        src = s_; dst = d_; bytes = n; pending = STAGE_THREADS; generation++;
        cv_work.notify_all();
        cv_done.wait(lk, [&] { return pending == 0; });
    }
    // host -> device copy of `n` bytes on `st`, staged block by block; returns when the LAST block has been queued
    cudaError_t copy(uint8_t* d_dev, const uint8_t* h_src, size_t n, cudaStream_t st) {
        for (size_t off = 0; off < n; off += STAGE_BLOCK) {
            const int k = (int)(next++ % STAGE_SLOTS);
            if (used[k]) {
                cudaError_t e = cudaEventSynchronize(free_ev[k]);   // the DMA that read this block has finished
                if (e != cudaSuccess) return e;
            }
            const size_t len = std::min(STAGE_BLOCK, n - off);
            parallel_copy(slot[k], h_src + off, len);
            cudaError_t e = cudaMemcpyAsync(d_dev + off, slot[k], len, cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) e = cudaEventRecord(free_ev[k], st);
            if (e != cudaSuccess) return e;
            used[k] = true;
        }
        return cudaSuccess;
    }
    void shutdown() {
        if (!ok) return;
        { std::lock_guard<std::mutex> g(mu); quit = true; }
        cv_work.notify_all();
        for (std::thread& w : workers) w.join();
        workers.clear();
        for (int i = 0; i < STAGE_SLOTS; i++) {
            if (free_ev[i]) cudaEventDestroy(free_ev[i]);
            if (slot[i]) cudaFreeHost(slot[i]);
            free_ev[i] = nullptr; slot[i] = nullptr; used[i] = false;
        }
        quit = false; ok = false;
    }
};
// heap-allocated and never destroyed: its worker threads must not meet a static destructor at process exit
// (lhb200_shutdown joins them and frees the ring)
KeyStager& g_stager = *new KeyStager;
std::mutex g_stager_use;   // one staged upload at a time (the ring is shared); concurrent big pageable uploads queue here

static bool host_pointer_is_pageable(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

std::mutex g_pool_mu;
std::vector<lhb200_bls_batch*> g_pool_free;
constexpr size_t POOL_MAX_IDLE = 64;   // idle handles kept (a 64-set handle is ~0.5 MB of device memory)

lhb200_bls_batch* pool_acquire(uint32_t n_sets, uint64_t n_keys) {
    lhb200_bls_batch* b = nullptr;
    {
        std::lock_guard<std::mutex> g(g_pool_mu);
        // best fit: the smallest idle handle that is large enough
        size_t best = SIZE_MAX;
        for (size_t i = 0; i < g_pool_free.size(); i++) {
            lhb200_bls_batch* c = g_pool_free[i];
            if (c->cap_sets >= n_sets && c->cap_keys >= n_keys &&
                (best == SIZE_MAX || c->cap_keys < g_pool_free[best]->cap_keys)) best = i;
        }
        if (best != SIZE_MAX) {
            b = g_pool_free[best];
            g_pool_free.erase(g_pool_free.begin() + best);
        } else if (g_pool_free.size() >= POOL_MAX_IDLE) {   // recycle the oldest handle's slot
            lhb200_bls_batch* victim = g_pool_free.front();
            g_pool_free.erase(g_pool_free.begin());
            cudaStreamSynchronize(victim->s_main);
            batch_free(victim);
        }
    }
    if (b) return b;
    const uint32_t cap_sets = std::max<uint32_t>(n_sets + n_sets / 4, 256);
    const uint64_t cap_keys = std::max<uint64_t>(n_keys + n_keys / 4, 4096);
    if (lhb200_bls_batch_create(cap_sets, cap_keys, &b) != LHB200_OK) return nullptr;
    return b;
}
void pool_release(lhb200_bls_batch* b) {
    std::lock_guard<std::mutex> g(g_pool_mu);
    g_pool_free.push_back(b);
}
}  // namespace
namespace lhb200 {
void bls_shutdown() {
    g_stager.shutdown();
    std::lock_guard<std::mutex> g(g_pool_mu);
    for (lhb200_bls_batch* b : g_pool_free) batch_free(b);
    g_pool_free.clear();
}
}  // namespace lhb200

extern "C" {

int32_t lhb200_bls_batch_create(uint32_t max_sets, uint64_t max_keys, lhb200_bls_batch** out) {
    LHB_REQUIRE_READY();
    if (!out || max_sets == 0) { set_error("bls_batch_create: bad arguments"); return LHB200_EINVAL; }
    lhb200_bls_batch* b = new lhb200_bls_batch();
    b->cap_sets = max_sets;
    b->cap_keys = max_keys;
    // sum-tree buffers: sized for the narrowest chunk in use (4 points per warp in latency mode, REDUCE_CHUNK otherwise)
    const uint64_t n = max_sets, n1 = cdiv(n, 4) + 1, n2 = cdiv(n1, 4) + 1;
    // Miller values: one per set (old kernels) or 5 per warp of the cooperative kernel (<= ceil((n+1)/6) + 40 warps)
    const uint64_t nf = std::max<uint64_t>(n, (cdiv(n + 1, 6) + 48) * 5), nf1 = cdiv(nf, REDUCE_CHUNK) + 1,
                   nf2 = cdiv(nf1, REDUCE_CHUNK) + 1;
#define ALLOC(p, bytes)                                                         \
    do {                                                                        \
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&(p)), (bytes));    \
        if (e != cudaSuccess) { batch_free(b); return cuda_fail(e, "cudaMalloc(" #p ")"); } \
    } while (0)
    ALLOC(b->d_sigs, n * 96 + 16);
    ALLOC(b->d_msgs, n * 32 + 16);
    ALLOC(b->d_pks, std::max<uint64_t>(max_keys, 1) * 96 + 16);
    ALLOC(b->d_offsets, (n + 1) * 4);
    ALLOC(b->d_rands, n * 8);
    ALLOC(b->d_sigr, n * sizeof(G2Jac));
    ALLOC(b->d_sig_tmp[0], n1 * sizeof(G2Jac));
    ALLOC(b->d_sig_tmp[1], n2 * sizeof(G2Jac));
    ALLOC(b->d_p, n * sizeof(G1Proj3));
    ALLOC(b->d_h, n * sizeof(G2Jac));
    ALLOC(b->d_f, nf * sizeof(Fp12));
    ALLOC(b->d_f_tmp[0], nf1 * sizeof(Fp12));
    ALLOC(b->d_f_tmp[1], nf2 * sizeof(Fp12));
    ALLOC(b->d_flast, sizeof(Fp12));
    ALLOC(b->d_gt, sizeof(Fp12));
    ALLOC(b->d_status, n);
    ALLOC(b->d_pk_status, n);
    ALLOC(b->d_fail, 4);
    ALLOC(b->d_ok, 4);
    ALLOC(b->d_neg_g1, sizeof(G1Proj3));
    ALLOC(b->d_pk_part, std::min<uint64_t>(n, PK_SPLIT_MAX_SETS) * PK_SLICES * sizeof(G1Jac));
    ALLOC(b->d_pk_part_bad, std::min<uint64_t>(n, PK_SPLIT_MAX_SETS) * PK_SLICES);
    ALLOC(b->d_members, n * 4);
    ALLOC(b->d_goffsets, (n + 1) * 4);
    ALLOC(b->d_gmsgs, n * 32 + 16);
    ALLOC(b->d_gp, n * sizeof(G1Proj3));
    ALLOC(b->d_gskip, n);
    ALLOC(b->d_gtmp, n * sizeof(G1Jac));
#undef ALLOC
    b->grouper.reserve(max_sets);
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&b->h_res), 2 * n + 64 + sizeof(Fp12), cudaHostAllocDefault);
    if (e != cudaSuccess) { batch_free(b); return cuda_fail(e, "cudaHostAlloc(result)"); }
    if ((e = cudaStreamCreateWithFlags(&b->s_main, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&b->s2, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&b->s3, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_h2c, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_sig, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_fork, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_join, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreate(&b->e_k0)) != cudaSuccess || (e = cudaEventCreate(&b->e_k1)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_done, cudaEventBlockingSync | cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_small, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->e_copy_free, cudaEventDisableTiming)) != cudaSuccess) {
        batch_free(b);
        return cuda_fail(e, "stream/event create");
    }
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // the key chunks must not queue behind the 1563-CTA kernels
    for (int j = 0; j < lhb200_bls_batch::N_PK_STREAMS; j++)
        if ((e = cudaStreamCreateWithPriority(&b->s_pk[j], cudaStreamNonBlocking, prio_hi)) != cudaSuccess ||
            (e = cudaEventCreateWithFlags(&b->e_pk[j], cudaEventDisableTiming)) != cudaSuccess) {
            batch_free(b);
            return cuda_fail(e, "stream create");
        }
    k_init_neg_g1<<<1, 32, 0, b->s_main>>>(b->d_neg_g1);
    if ((e = cudaStreamSynchronize(b->s_main)) != cudaSuccess) { batch_free(b); return cuda_fail(e, "k_init_neg_g1"); }
    *out = b;
    return LHB200_OK;
}

int32_t lhb200_bls_batch_destroy(lhb200_bls_batch* b) {
    if (ctx().ready) cudaDeviceSynchronize();
    batch_free(b);
    return LHB200_OK;
}

// ---- blinding scalars (blst.rs:46-68: `rand::thread_rng()`, a ChaCha CSPRNG seeded from the OS) ----------------
// Same construction: a ChaCha20 keystream (RFC 8439 block function) keyed with 256 bits from getrandom(2) per thread,
// re-keyed every 2^20 blocks; every 64-bit word is used as one scalar, zeros are skipped (blst.rs:60-64).
namespace {
struct ChaChaRng {
    uint32_t key[8];
    uint32_t nonce[3];
    uint32_t counter = 0;
    bool keyed = false;
    uint64_t buf[8];
    int have = 0;
    static inline uint32_t rotl(uint32_t v, int c) { return (v << c) | (v >> (32 - c)); }
    static inline void qr(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
        a += b; d ^= a; d = rotl(d, 16);
        c += d; b ^= c; b = rotl(b, 12);
        a += b; d ^= a; d = rotl(d, 8);
        c += d; b ^= c; b = rotl(b, 7);
    }
    bool rekey() {
        uint8_t seed[44];
        size_t got = 0;
        while (got < sizeof seed) {
            const ssize_t k = getrandom(seed + got, sizeof seed - got, 0);
            if (k < 0) { if (errno == EINTR) continue; return false; }
            got += (size_t)k;
        }
        memcpy(key, seed, 32);
        memcpy(nonce, seed + 32, 12);
        counter = 0;
        keyed = true;
        return true;
    }
    bool refill() {
        if (!keyed || counter >= (1u << 20)) { if (!rekey()) return false; }
        uint32_t st[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
                           key[4], key[5], key[6], key[7], counter, nonce[0], nonce[1], nonce[2]};
        uint32_t x[16];
        memcpy(x, st, sizeof x);
        for (int i = 0; i < 10; i++) {
            qr(x[0], x[4], x[8], x[12]); qr(x[1], x[5], x[9], x[13]); qr(x[2], x[6], x[10], x[14]); qr(x[3], x[7], x[11], x[15]);
            qr(x[0], x[5], x[10], x[15]); qr(x[1], x[6], x[11], x[12]); qr(x[2], x[7], x[8], x[13]); qr(x[3], x[4], x[9], x[14]);
        }
        for (int i = 0; i < 16; i++) x[i] += st[i];
        memcpy(buf, x, sizeof buf);
        counter++;
        have = 8;
        return true;
    }
    bool next(uint64_t& v) {
        do {
            if (have == 0 && !refill()) return false;
            v = buf[--have];
        } while (v == 0);
        return true;
    }
};
}  // namespace
static bool gen_rands(uint64_t* r, uint32_t n) {
    static thread_local ChaChaRng rng;
    for (uint32_t i = 0; i < n; i++)
        if (!rng.next(r[i])) return false;
    return true;
}
// Test hook: n scalars from the generator above (statistical / distinctness tests without a device).
extern "C" LHB200_API int32_t lhb200_debug_rand_scalars(uint64_t* out, uint32_t n) {
    if (!out) return LHB200_EINVAL;
    return gen_rands(out, n) ? LHB200_OK : LHB200_ECUDA;
}

// Test hook: the grouping lhb200_bls_batch_upload* applies to the messages (no device needed).
extern "C" LHB200_API int32_t lhb200_debug_group_messages(const uint8_t* msgs, uint32_t n, uint32_t* members,
                                                          uint32_t* group_offsets, uint32_t* n_groups) {
    if (!msgs || !members || !group_offsets || !n_groups) return LHB200_EINVAL;
    MsgGrouper g;
    g.reserve(n);
    uint32_t max_group = 0;
    const uint32_t ng = g.run(msgs, n, 0, &max_group);
    memcpy(members, g.members.data(), (size_t)n * 4);
    memcpy(group_offsets, g.offsets.data(), (size_t)(ng + 1) * 4);
    *n_groups = ng;
    return LHB200_OK;
}

// Grouping is used once at least 1/GROUP_MIN_REPEAT_DIV of the sets repeat a message.  Measured on one H100 80GB HBM3
// at 700 W (DESIGN §2.6): 100 000 x 128-key sets with one repeated message lost ~4.5 ms per plugin call to grouping
// (host CSR, copies, group-sum tree), while 97 952 repeats saved ~49 ms of hash-to-G2 and Miller work (~0.5 us each).
constexpr uint32_t GROUP_MIN_REPEAT_DIV = 8;

// Host uploads: group the sets by message and queue the CSR and the distinct messages on `s`.  n_groups stays 0 (the
// ungrouped path) when too few messages repeat, or with LHB_GROUP_MESSAGES=0.
// Segmented pass: the same policy over the whole pass, with (segment, message) as the group key.  Each segment is grouped
// on its own and the CSRs are concatenated, so a group never spans two segments and a segment's groups (its pairs) stay
// contiguous.  Queues the set and pair offsets of the segments on `s`.
static int32_t upload_segment_groups(lhb200_bls_batch* b, const uint8_t* msgs, uint32_t n, cudaStream_t s) {
    const uint32_t K = b->n_seg;
    uint32_t* set_off = b->seg_h.data();
    uint32_t* pair_off = set_off + K + 1;
    memcpy(pair_off, set_off, (size_t)(K + 1) * 4);
    if (g_cfg.group_messages && n >= 2) {
        MsgGrouper& g = b->grouper;
        b->seg_members.resize(n);
        b->seg_goffsets.resize(n + 1);
        b->seg_gmsgs.resize((size_t)n * 32);
        uint32_t ng = 0, max_group = 0;
        b->seg_goffsets[0] = 0;
        for (uint32_t k = 0; k < K; k++) {
            const uint32_t lo = set_off[k], m = set_off[k + 1] - lo;
            uint32_t mg = 0;
            const uint32_t gk = g.run(msgs + (size_t)32 * lo, m, 0, &mg);
            for (uint32_t i = 0; i < m; i++) b->seg_members[lo + i] = lo + g.members[i];
            for (uint32_t j = 0; j < gk; j++) b->seg_goffsets[ng + j + 1] = lo + g.offsets[j + 1];
            memcpy(&b->seg_gmsgs[(size_t)32 * ng], g.msgs.data(), (size_t)32 * gk);
            ng += gk;
            max_group = std::max(max_group, mg);
            pair_off[k + 1] = ng;
        }
        if (n - ng >= std::max<uint32_t>(1, n / GROUP_MIN_REPEAT_DIV)) {
            LHB_CUDA(cudaMemcpyAsync(b->d_members, b->seg_members.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
            LHB_CUDA(cudaMemcpyAsync(b->d_goffsets, b->seg_goffsets.data(), (size_t)(ng + 1) * 4, cudaMemcpyHostToDevice, s));
            LHB_CUDA(cudaMemcpyAsync(b->d_gmsgs, b->seg_gmsgs.data(), (size_t)ng * 32, cudaMemcpyHostToDevice, s));
            b->n_groups = ng;
            b->max_group = max_group;
        } else {
            memcpy(pair_off, set_off, (size_t)(K + 1) * 4);
        }
    }
    LHB_CUDA(cudaMemcpyAsync(b->d_seg_off, set_off, (size_t)2 * (K + 1) * 4, cudaMemcpyHostToDevice, s));
    return LHB200_OK;
}

static int32_t upload_groups(lhb200_bls_batch* b, const uint8_t* msgs, uint32_t n, cudaStream_t s) {
    b->n_groups = 0;
    if (b->n_seg) return upload_segment_groups(b, msgs, n, s);
    if (!g_cfg.group_messages || n < 2) return LHB200_OK;
    MsgGrouper& g = b->grouper;
    const uint32_t min_repeats = std::max<uint32_t>(1, n / GROUP_MIN_REPEAT_DIV);
    const uint32_t ng = g.run(msgs, n, min_repeats, &b->max_group);
    if (n - ng < min_repeats) return LHB200_OK;
    LHB_CUDA(cudaMemcpyAsync(b->d_members, g.members.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaMemcpyAsync(b->d_goffsets, g.offsets.data(), (size_t)(ng + 1) * 4, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaMemcpyAsync(b->d_gmsgs, g.msgs.data(), (size_t)ng * 32, cudaMemcpyHostToDevice, s));
    b->n_groups = ng;
    return LHB200_OK;
}

// What the three host uploads share.  Checks the arguments, draws the scalars into b->rbuf when rands is NULL (or
// rejects a zero one), queues the copies of the signatures, messages, offsets and scalars and the message grouping on
// `s`, and binds the batch's own buffers as its inputs.  `keys` is the key buffer (at most cap_keys keys) or, with a
// table, the key indices; the caller copies them.
static int32_t stage_inputs(const char* fn, lhb200_bls_batch* b, const lhb200_pubkey_table* table, const uint8_t* sigs,
                            const uint8_t* msgs, const void* keys, const uint32_t* pk_offsets, const uint64_t* rands,
                            uint32_t n_sets, cudaStream_t s) {
    if (!b || n_sets == 0 || n_sets > b->cap_sets || !sigs || !msgs || !pk_offsets) {
        set_error("%s: bad arguments", fn);
        return LHB200_EINVAL;
    }
    const uint64_t n_keys = pk_offsets[n_sets];
    if (!table && n_keys > b->cap_keys) { set_error("%s: more keys than the batch holds", fn); return LHB200_EINVAL; }
    if (n_keys && !keys) { set_error("%s: no keys given", fn); return LHB200_EINVAL; }
    for (uint32_t i = 0; i < n_sets; i++)
        if (pk_offsets[i] > pk_offsets[i + 1]) { set_error("%s: offsets not monotone", fn); return LHB200_EINVAL; }
    if (b->n_seg && b->seg_h[b->n_seg] != n_sets) {
        set_error("%s: the segments cover %u sets, not %u", fn, b->seg_h[b->n_seg], n_sets);
        return LHB200_EINVAL;
    }
    if (!rands) {
        b->rbuf.resize(n_sets);
        if (!gen_rands(b->rbuf.data(), n_sets)) { set_error("%s: getrandom(2) failed", fn); return LHB200_ECUDA; }
        rands = b->rbuf.data();
    } else {
        for (uint32_t i = 0; i < n_sets; i++)
            if (rands[i] == 0) { set_error("%s: zero random scalar", fn); return LHB200_EINVAL; }
    }
    LHB_CUDA(cudaMemcpyAsync(b->d_sigs, sigs, (size_t)n_sets * 96, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaMemcpyAsync(b->d_msgs, msgs, (size_t)n_sets * 32, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaMemcpyAsync(b->d_offsets, pk_offsets, (size_t)(n_sets + 1) * 4, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaMemcpyAsync(b->d_rands, rands, (size_t)n_sets * 8, cudaMemcpyHostToDevice, s));
    if (int32_t rc = upload_groups(b, msgs, n_sets, s)) return rc;
    b->n = n_sets;
    b->n_chunks = 0;
    b->in_sigs = b->d_sigs; b->in_msgs = b->d_msgs; b->in_pks = table ? nullptr : b->d_pks;
    b->in_offsets = b->d_offsets; b->in_rands = b->d_rands;
    b->table = table;
    return LHB200_OK;
}

// Copy host inputs into the batch's device buffers.  rands == NULL: drawn here.
int32_t lhb200_bls_batch_upload(lhb200_bls_batch* b, const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets) {
    LHB_REQUIRE_READY();
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    if (int32_t rc = stage_inputs("bls_batch_upload", b, nullptr, sigs, msgs, pks, pk_offsets, rands, n_sets, c.stream))
        return rc;
    const uint64_t n_keys = pk_offsets[n_sets];
    if (n_keys) LHB_CUDA(cudaMemcpyAsync(b->d_pks, pks, (size_t)n_keys * 96, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));  // caller buffers may go away
    return LHB200_OK;
}

// Streamed form of lhb200_bls_batch_upload: queues the small arrays and BINDS the host key buffer; the key chunks are
// copied by lhb200_bls_batch_verify_enqueue, interleaved with their aggregation kernels.  The host buffers must stay
// valid and unchanged until lhb200_bls_batch_result returns.  The small arrays go first; the keys (96 B x K, 1.2 GB at
// 100 k x 128) follow in chunks of whole sets on a copy stream, and lhb200_bls_batch_verify_enqueue aggregates each
// chunk as it lands while k_sig_prepare / k_hash_to_g2 already run — the host link hides behind the ALU-bound kernels.
int32_t lhb200_bls_batch_upload_async(lhb200_bls_batch* b, const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                      const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets, void* stream) {
    LHB_REQUIRE_READY();
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    if (int32_t rc = stage_inputs("bls_batch_upload_async", b, nullptr, sigs, msgs, pks, pk_offsets, rands, n_sets, s))
        return rc;
    // the previous verify on this batch may still be reading d_pks: order the new copies behind it
    LHB_CUDA(cudaEventRecord(b->e_copy_free, s));
    for (cudaStream_t st : b->s_pk) LHB_CUDA(cudaStreamWaitEvent(st, b->e_copy_free, 0));
    LHB_CUDA(cudaEventRecord(b->e_small, s));
    // chunks of whole sets, ~equal key counts
    const uint64_t n_keys = pk_offsets[n_sets];
    int nc = (int)std::min<uint64_t>(lhb200_bls_batch::MAX_CHUNKS, std::max<uint64_t>(1, n_keys * 96 / (32u << 20)));
    nc = std::min<int>(nc, (int)n_sets);
    b->chunk_lo[0] = 0;
    uint32_t lo = 0;
    for (int c = 0; c < nc; c++) {
        uint32_t hi;
        if (c == nc - 1) hi = n_sets;
        else {
            const uint64_t target = n_keys * (uint64_t)(c + 1) / nc;
            hi = (uint32_t)(std::lower_bound(pk_offsets + lo, pk_offsets + n_sets + 1, target) - pk_offsets);
            hi = std::min<uint32_t>(std::max<uint32_t>(hi, lo), n_sets);
        }
        b->chunk_key[c] = pk_offsets[lo];
        b->chunk_key[c + 1] = pk_offsets[hi];
        b->chunk_lo[c + 1] = hi;
        lo = hi;
    }
    b->n_chunks = nc;
    b->h_pks = pks;
    return LHB200_OK;
}

// ---- device-resident pubkey table (SURVEY §8f-1; mirror of ValidatorPubkeyCache) ---------------------------
int32_t lhb200_pubkey_table_create(uint64_t capacity, lhb200_pubkey_table** out) {
    LHB_REQUIRE_READY();
    if (!out || capacity == 0) return LHB200_EINVAL;
    lhb200_pubkey_table* t = new lhb200_pubkey_table();
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&t->d_keys), capacity * sizeof(G1Mont));
    if (e != cudaSuccess) { delete t; return cuda_fail(e, "cudaMalloc(pubkey table)"); }
    t->capacity = capacity;
    *out = t;
    return LHB200_OK;
}
int32_t lhb200_pubkey_table_destroy(lhb200_pubkey_table* t) {
    if (!t) return LHB200_OK;
    if (ctx().ready) cudaDeviceSynchronize();
    if (t->d_keys) cudaFree(t->d_keys);
    delete t;
    return LHB200_OK;
}
uint64_t lhb200_pubkey_table_len(const lhb200_pubkey_table* t) { return t ? t->len : 0; }

// Append n validated keys (96-byte uncompressed, the validator_pubkey_cache.rs:195-199 format) at indices
// [len, len+n).  Malformed / off-curve / infinity entries make the call fail with LHB200_EDECODE (nothing appended).
int32_t lhb200_pubkey_table_append(lhb200_pubkey_table* t, const uint8_t* pks96, uint64_t n) {
    LHB_REQUIRE_READY();
    if (!t || (n && !pks96)) return LHB200_EINVAL;
    if (t->len + n > t->capacity) { set_error("pubkey table full"); return LHB200_EINVAL; }
    if (n == 0) return LHB200_OK;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(n * 96 + 256));
    if (!d) return LHB200_ENOMEM;
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(d + ((n * 96 + 15) / 16) * 16);
    LHB_CUDA(cudaMemcpyAsync(d, pks96, n * 96, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemsetAsync(d_bad, 0, 4, c.stream));
    k_table_import<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, (uint32_t)n, t->d_keys + t->len, d_bad);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    uint32_t bad = 0;
    LHB_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    if (bad) { set_error("%u of %llu keys are malformed, off-curve or at infinity", bad, (unsigned long long)n); return LHB200_EDECODE; }
    t->len += n;
    return LHB200_OK;
}

// Like lhb200_bls_batch_upload, but the signing keys are given as indices into a resident table
// (what signature_sets.rs:315-320 gathers from the pubkey cache): key_indices[K], CSR offsets as before.
int32_t lhb200_bls_batch_upload_indexed(lhb200_bls_batch* b, const lhb200_pubkey_table* table, const uint8_t* sigs,
                                        const uint8_t* msgs, const uint32_t* key_indices, const uint32_t* pk_offsets,
                                        const uint64_t* rands, uint32_t n_sets) {
    LHB_REQUIRE_READY();
    if (!table) { set_error("bls_batch_upload_indexed: no pubkey table"); return LHB200_EINVAL; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    cudaStream_t s = c.stream;
    if (int32_t rc = stage_inputs("bls_batch_upload_indexed", b, table, sigs, msgs, key_indices, pk_offsets, rands, n_sets, s))
        return rc;
    const uint64_t n_keys = pk_offsets[n_sets];
    if (n_keys > b->cap_indices) {
        b->n = 0;   // no inputs until the indices have a buffer
        if (b->d_indices) { cudaStreamSynchronize(s); cudaFree(b->d_indices); b->d_indices = nullptr; b->cap_indices = 0; }
        LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&b->d_indices), std::max<uint64_t>(n_keys, 1) * 4));
        b->cap_indices = n_keys;
        b->n = n_sets;
    }
    if (n_keys) LHB_CUDA(cudaMemcpyAsync(b->d_indices, key_indices, (size_t)n_keys * 4, cudaMemcpyHostToDevice, s));
    LHB_CUDA(cudaStreamSynchronize(s));
    return LHB200_OK;
}

// Use caller-owned device buffers (16-byte aligned) as the inputs: nothing is copied.
int32_t lhb200_bls_batch_set_device_inputs(lhb200_bls_batch* b, const void* d_sigs, const void* d_msgs,
                                           const void* d_pks, const void* d_offsets, const void* d_rands,
                                           uint32_t n_sets) {
    LHB_REQUIRE_READY();
    if (!b || n_sets == 0 || n_sets > b->cap_sets || !d_sigs || !d_msgs || !d_offsets || !d_rands ||
        ((uintptr_t)d_sigs & 15) || ((uintptr_t)d_msgs & 15) || ((uintptr_t)d_pks & 15)) {
        set_error("bls_batch_set_device_inputs: bad arguments (buffers must be 16-byte aligned)");
        return LHB200_EINVAL;
    }
    b->n = n_sets;
    b->in_sigs = static_cast<const uint8_t*>(d_sigs);
    b->in_msgs = static_cast<const uint8_t*>(d_msgs);
    b->in_pks = static_cast<const uint8_t*>(d_pks);
    b->in_offsets = static_cast<const uint32_t*>(d_offsets);
    b->in_rands = static_cast<const uint64_t*>(d_rands);
    b->n_chunks = 0;
    b->n_groups = 0;   // device-resident messages are not grouped
    b->n_seg = 0;      // segments apply to the host uploads only
    b->table = nullptr;
    return LHB200_OK;
}

// ---- verify_enqueue: one launch helper per stage, following the Plan ------------------------------------------
// s2: r_i sig_i, their sum tree and, with k_miller_multi, the pair (-g1, sum r sig) on its own
static int32_t launch_signatures(lhb200_bls_batch* b, const Plan& p, uint64_t& launches) {
    const uint32_t n = b->n, *w = p.w;
    const size_t gw_smem = gw::smem_bytes(GW_WPB);
    if (w[LHB200_PLAN_SIG] == LHB200_K_SIG_PREPARE_WARP)
        gw::k_sig_prepare_warp<<<cdiv(n, GW_WPB), 32 * GW_WPB, gw_smem, b->s2>>>(b->in_sigs, b->in_rands, n, b->d_sigr,
                                                                               b->d_status, b->d_fail);
    else
        k_sig_prepare<<<w[LHB200_PLAN_LANE_GRID], BLS_BLOCK, 0, b->s2>>>(b->in_sigs, b->in_rands, n, b->d_sigr, b->d_status,
                                                                        b->d_fail);
    LHB_CUDA(cudaEventRecord(b->e_sig, b->s2));
    if (w[LHB200_PLAN_SEGMENTS]) {   // one sum per segment, in place over the set positions
        uint64_t span = 1;
        for (uint32_t level = 0; level < w[LHB200_PLAN_SUM_LEVELS]; level++, span *= GROUP_CHUNK)
            k_g2_segment_sum<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, b->s2>>>(b->d_sigr, b->d_seg_off, n, w[LHB200_PLAN_SEGMENTS],
                                                                           level, span, b->d_seg_sig);
        b->d_sig_sum = b->d_seg_sig;
        launches += 1 + w[LHB200_PLAN_SUM_LEVELS];
        LHB_CUDA(cudaEventRecord(b->e_join, b->s2));
        return LHB200_OK;
    }
    const bool warp = w[LHB200_PLAN_SUM] == LHB200_K_G2_SUM_WARP;   // latency mode: warp-wide additions
    b->d_sig_sum = reduce_tree(b->d_sigr, n, warp ? G2_SUM_WARP_CHUNK : REDUCE_CHUNK, w[LHB200_PLAN_SUM_LEVELS], b->d_sig_tmp,
                               [&](const G2Jac* in, uint32_t m, uint32_t mo, G2Jac* out) {
                                   if (warp)
                                       gw::k_g2_sum_warp<<<cdiv(mo, GW_WPB), 32 * GW_WPB, gw_smem, b->s2>>>(in, m, G2_SUM_WARP_CHUNK, out);
                                   else
                                       k_g2_reduce<<<cdiv(mo, BLS_BLOCK), BLS_BLOCK, 0, b->s2>>>(in, m, REDUCE_CHUNK, out);
                               });
    launches += 1 + w[LHB200_PLAN_SUM_LEVELS];
    if (w[LHB200_PLAN_LAST_MILLER]) {
        k_last_miller<<<1, 32, 0, b->s2>>>(b->d_sig_sum, b->d_flast);
        launches++;
    }
    LHB_CUDA(cudaEventRecord(b->e_join, b->s2));
    return LHB200_OK;
}

// s3: H(m_i), or H(message of group g) in a grouped batch
static int32_t launch_hash(lhb200_bls_batch* b, const Plan& p, uint64_t& launches) {
    const uint8_t* msgs = b->n_groups ? b->d_gmsgs : b->in_msgs;
    switch (p.w[LHB200_PLAN_HASH]) {
    case LHB200_K_HASH_TO_G2_WARP:
        gw::k_hash_to_g2_warp<<<p.hash_grid, 32 * GW_WPB, gw::smem_bytes(GW_WPB), b->s3>>>(msgs, p.ng, b->d_h);
        break;
    case LHB200_K_HASH_TO_G2_PAIR: k_hash_to_g2_pair<<<p.hash_grid, BLS_BLOCK, 0, b->s3>>>(msgs, p.ng, b->d_h); break;
    default: k_hash_to_g2<<<p.hash_grid, BLS_BLOCK, 0, b->s3>>>(msgs, p.ng, b->d_h);
    }
    launches++;
    LHB_CUDA(cudaEventRecord(b->e_h2c, b->s3));
    return LHB200_OK;
}

// r_i apk_i: from the pubkey table or the key buffer on s, or, after a streamed upload, chunk by chunk on the
// (high-priority) stream that copies the chunk, as soon as its keys have landed
static int32_t launch_keys(lhb200_bls_batch* b, const Plan& p, cudaStream_t s, uint64_t& launches) {
    const uint32_t key = p.w[LHB200_PLAN_KEY], grid = p.w[LHB200_PLAN_LANE_GRID];
    if (key == LHB200_K_PK_AGGREGATE_INDEXED) {
        k_pk_aggregate_indexed<<<grid, BLS_BLOCK, 0, s>>>(b->table->d_keys, (uint32_t)b->table->len, b->d_indices,
                                                         b->in_offsets, b->in_rands, b->n, b->d_p, b->d_pk_status, b->d_fail);
        launches++;
        return LHB200_OK;
    }
    auto launch_pk = [&](uint32_t lo, uint32_t cnt, cudaStream_t st) {   // sets [lo, lo + cnt)
        if (key == LHB200_K_PK_AGGREGATE_TMA) {
            k_pk_aggregate_tma<<<cdiv(cnt, BLS_BLOCK), BLS_BLOCK, 0, st>>>(b->in_pks, b->in_offsets + lo, b->in_rands + lo, cnt,
                                                                          b->d_p + lo, b->d_pk_status + lo, b->d_fail);
        } else if (key == LHB200_K_PK_PARTIAL_COMBINE) {
            k_pk_partial<<<cdiv(cnt * PK_SLICES, BLS_BLOCK), BLS_BLOCK, 0, st>>>(
                b->in_pks, b->in_offsets + lo, cnt, b->d_pk_part + (size_t)lo * PK_SLICES, b->d_pk_part_bad + (size_t)lo * PK_SLICES);
            k_pk_combine<<<cdiv(cnt, BLS_BLOCK), BLS_BLOCK, 0, st>>>(
                b->d_pk_part + (size_t)lo * PK_SLICES, b->d_pk_part_bad + (size_t)lo * PK_SLICES, b->in_offsets + lo,
                b->in_rands + lo, cnt, b->d_p + lo, b->d_pk_status + lo, b->d_fail);
            launches++;
        } else {
            k_pk_aggregate<<<std::min<uint32_t>(grid, cdiv(cnt, BLS_BLOCK)), BLS_BLOCK, 0, st>>>(
                b->in_pks, b->in_offsets + lo, b->in_rands + lo, cnt, b->d_p + lo, b->d_pk_status + lo, b->d_fail);
        }
        launches++;
    };
    if (!b->n_chunks) {
        launch_pk(0, b->n, s);
        return LHB200_OK;
    }
    // big pageable key buffers go through the library's pinned ring (see KeyStager)
    const uint64_t key_bytes = (b->chunk_key[b->n_chunks] - b->chunk_key[0]) * 96;
    std::unique_lock<std::mutex> stage_lock(g_stager_use, std::defer_lock);
    bool stage_keys = false;
    if (g_cfg.stage_pageable && key_bytes >= STAGE_MIN_BYTES && host_pointer_is_pageable(b->h_pks)) {
        stage_lock.lock();
        stage_keys = g_stager.init();
        if (!stage_keys) stage_lock.unlock();
    }
    for (int j = 0; j < lhb200_bls_batch::N_PK_STREAMS; j++) LHB_CUDA(cudaStreamWaitEvent(b->s_pk[j], b->e_fork, 0));
    for (int c = 0; c < b->n_chunks; c++) {
        const uint32_t lo = b->chunk_lo[c], cnt = b->chunk_lo[c + 1] - lo;
        const uint64_t k0 = b->chunk_key[c], k1 = b->chunk_key[c + 1];
        cudaStream_t st = b->s_pk[c % lhb200_bls_batch::N_PK_STREAMS];
        if (k1 > k0) {
            if (stage_keys) LHB_CUDA(g_stager.copy(b->d_pks + k0 * 96, b->h_pks + k0 * 96, (k1 - k0) * 96, st));
            else LHB_CUDA(cudaMemcpyAsync(b->d_pks + k0 * 96, b->h_pks + k0 * 96, (k1 - k0) * 96, cudaMemcpyHostToDevice, st));
        }
        if (cnt) launch_pk(lo, cnt, st);
    }
    for (int j = 0; j < lhb200_bls_batch::N_PK_STREAMS; j++) {
        LHB_CUDA(cudaEventRecord(b->e_pk[j], b->s_pk[j]));
        LHB_CUDA(cudaStreamWaitEvent(s, b->e_pk[j], 0));
    }
    return LHB200_OK;
}

// Grouped batches: per group, the sum of r_i apk_i over its contributing members, and a skip flag
static void launch_group_sum(lhb200_bls_batch* b, const Plan& p, cudaStream_t s, uint64_t& launches) {
    GroupSumArgs ga;
    ga.P = b->d_p; ga.status = b->d_status; ga.pk_status = b->d_pk_status;
    ga.members = b->d_members; ga.offsets = b->d_goffsets; ga.n = b->n; ga.n_groups = p.ng;
    ga.tmp = b->d_gtmp; ga.out_p = b->d_gp; ga.skip = b->d_gskip;
    const uint32_t levels = p.w[LHB200_PLAN_GROUP_SUM_LEVELS];
    uint64_t span = 1;
    for (uint32_t level = 0; level < levels; level++, span *= GROUP_CHUNK)
        k_g1_group_sum<<<cdiv(b->n, BLS_BLOCK), BLS_BLOCK, 0, s>>>(ga, level, span);
    launches += levels;
}

// The Miller kernel between e_k0 and e_k1, then the product tree down to the final kernel's tail (-> *prod).  The
// kernels pair (P[i], d_h[i]), i < ng, and skip i unless st[i] | pk_st[i] == 0: per set, or per group (the group sums,
// with the skip flag in both status slots).
static int32_t launch_miller(lhb200_bls_batch* b, const Plan& p, cudaStream_t s, uint64_t& launches, const Fp12** prod) {
    const uint32_t* w = p.w;
    const bool grouped = b->n_groups != 0, multi = w[LHB200_PLAN_MILLER] == LHB200_K_MILLER_MULTI;
    const G1Proj3* P = grouped ? b->d_gp : b->d_p;
    const uint8_t* st = grouped ? b->d_gskip : b->d_status;
    const uint8_t* pk_st = grouped ? b->d_gskip : b->d_pk_status;
    const uint32_t grid = w[LHB200_PLAN_MILLER_GRID], wpb = w[LHB200_PLAN_MILLER_WPB];
    const uint32_t n_seg = w[LHB200_PLAN_SEGMENTS];
    Fp12* const f = n_seg ? b->d_seg_f : b->d_f;
    if (!multi) LHB_CUDA(cudaStreamWaitEvent(s, b->e_join, 0));   // sum r sig (and -g1) ready
    LHB_CUDA(cudaEventRecord(b->e_k0, s));
    if (n_seg)
        mw::k_miller_warp_segments<<<grid, 32 * wpb, mw::smem_bytes((int)wpb), s>>>(P, b->d_h, st, pk_st, p.ng, b->d_seg_sig,
                                                                                  n_seg, b->d_neg_g1, f);
    else if (w[LHB200_PLAN_MILLER] == LHB200_K_MILLER_WARP)
        mw::k_miller_warp<<<grid, 32 * wpb, mw::smem_bytes((int)wpb), s>>>(P, b->d_h, st, pk_st, p.ng, b->d_sig_sum,
                                                                         b->d_neg_g1, b->d_f);
    else if (w[LHB200_PLAN_MILLER] == LHB200_K_MILLER_COOP)
        mc::k_miller_coop<<<grid, 32 * wpb, mc::mc_smem_bytes(), s>>>(P, b->d_h, st, pk_st, p.ng, b->d_sig_sum, b->d_neg_g1,
                                                                      w[LHB200_PLAN_MILLER_SPW], b->d_mc_scratch, b->d_f);
    else
        k_miller_multi<<<grid, MILLER_BLOCK, 0, s>>>(P, b->d_h, st, pk_st, p.ng, w[LHB200_PLAN_MILLER_SPW], p.miller_out,
                                                     b->d_f);
    LHB_CUDA(cudaEventRecord(b->e_k1, s));
    *prod = reduce_tree<Fp12>(f, p.miller_out, REDUCE_CHUNK, w[LHB200_PLAN_FP12_REDUCE_LEVELS], b->d_f_tmp,
                              [&](const Fp12* in, uint32_t m, uint32_t mo, Fp12* out) {
                                  k_fp12_reduce<<<cdiv(mo, BLS_BLOCK), BLS_BLOCK, 0, s>>>(in, m, REDUCE_CHUNK, out);
                              });
    launches += 1 + w[LHB200_PLAN_FP12_REDUCE_LEVELS];
    if (multi) LHB_CUDA(cudaStreamWaitEvent(s, b->e_join, 0));   // k_final_coop reads k_last_miller's value
    return LHB200_OK;
}

int32_t lhb200_bls_batch_verify_enqueue(lhb200_bls_batch* b, void* stream) {
    LHB_REQUIRE_READY();
    if (!b || b->n == 0 || !b->in_sigs) { set_error("bls_batch_verify_enqueue: no inputs"); return LHB200_EINVAL; }
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    const uint32_t n = b->n;
    const uint32_t n_seg = b->n_seg;
    if (n_seg && b->seg_h[n_seg] != n) { set_error("bls_batch_verify_enqueue: the segments do not cover the sets"); return LHB200_EINVAL; }
    const Plan p = choose(g_cfg, n, b->n_groups, b->max_group, b->table != nullptr, (uint32_t)b->n_chunks,
                          b->in_pks && ((uintptr_t)b->in_pks & 15) == 0, n_seg, b->max_seg);
    memcpy(b->plan, p.w, sizeof b->plan);
    if (p.mc_scratch_words > b->mc_scratch_words) {
        LHB_CUDA(cudaStreamSynchronize(s));
        if (b->d_mc_scratch) cudaFree(b->d_mc_scratch);
        b->d_mc_scratch = nullptr;
        LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&b->d_mc_scratch), p.mc_scratch_words * 4));
        b->mc_scratch_words = p.mc_scratch_words;
    }
    if (b->n_chunks) LHB_CUDA(cudaStreamWaitEvent(s, b->e_small, 0));  // streamed upload: small arrays first
    LHB_CUDA(cudaMemsetAsync(b->d_status, 0, n, s));
    LHB_CUDA(cudaMemsetAsync(b->d_fail, 0, 4, s));
    LHB_CUDA(cudaMemsetAsync(b->d_ok, 0, 4, s));
    // Three independent per-set stages run concurrently (they matter for small batches, where each kernel is a
    // latency-bound handful of warps): s2 = signatures, s3 = hash_to_g2, s = keys.  The Miller kernel joins all three.
    LHB_CUDA(cudaEventRecord(b->e_fork, s));
    LHB_CUDA(cudaStreamWaitEvent(b->s2, b->e_fork, 0));
    LHB_CUDA(cudaStreamWaitEvent(b->s3, b->e_fork, 0));
    uint64_t launches = 0;
    const Fp12* prod = nullptr;
    if (int32_t rc = launch_signatures(b, p, launches)) return rc;
    if (int32_t rc = launch_hash(b, p, launches)) return rc;
    if (int32_t rc = launch_keys(b, p, s, launches)) return rc;
    LHB_CUDA(cudaStreamWaitEvent(s, b->e_h2c, 0));
    LHB_CUDA(cudaStreamWaitEvent(s, b->e_sig, 0));    // the Miller kernel reads the status bytes k_sig_prepare may set
    if (b->n_groups) launch_group_sum(b, p, s, launches);
    if (int32_t rc = launch_miller(b, p, s, launches, &prod)) return rc;
    const uint32_t n_tail = p.w[LHB200_PLAN_N_TAIL];
    if (n_seg)   // one block per segment; pair offsets follow the set offsets in d_seg_off
        fe::k_final_segments<<<n_seg, 32 * fe::FE_WARPS, fe::smem_bytes(), s>>>(prod, p.ng, b->d_seg_off + n_seg + 1,
                                                                                b->d_seg_off, b->d_status, b->d_pk_status,
                                                                                b->d_seg_ok, b->d_seg_gt);
    else if (p.w[LHB200_PLAN_FINAL] == LHB200_K_FINAL_WARP)   // phase-interpreter tail (bls/fe_warp.cuh)
        fe::k_final_warp<<<1, 32 * fe::FE_WARPS, fe::smem_bytes(), s>>>(prod, n_tail, b->d_fail, b->d_ok, b->d_gt);
    else
        k_final_coop<<<1, COOP_THREADS, sizeof(CoopFinalSmem), s>>>(prod, n_tail, p.w[LHB200_PLAN_LAST_MILLER] ? b->d_flast : nullptr,
                                                                    b->d_fail, b->d_ok, b->d_gt);
    launches++;
    LHB_CUDA(cudaGetLastError());
    count_launch(launches);
    b->launches_last = launches;
    b->n_seg_last = n_seg;
    b->n_seg = 0;
    return LHB200_OK;
}

// ncclAllReduce(min) of the batch's device verdict over the library's communicator (lhb200_comm_init), enqueued on
// `stream` right behind lhb200_bls_batch_verify_enqueue: the one collective of the sharded BLS path (SURVEY.md §8e),
// on the device buffer, no host hop.  A no-op without a communicator.
int32_t lhb200_bls_batch_allreduce_verdict(lhb200_bls_batch* b, void* stream) {
    LHB_REQUIRE_READY();
    if (!b) return LHB200_EINVAL;
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    return comm_allreduce_min_u8(b->d_ok, 1, s);
}

// The verdicts (n_ok bytes at d_ok, through the pinned h_ok) and optionally the per-set statuses of the last verify.
static int32_t fetch_results(lhb200_bls_batch* b, cudaStream_t s, const uint8_t* d_ok, uint8_t* h_ok, uint32_t n_ok,
                             uint8_t* ok, uint8_t* set_status) {
    LHB_CUDA(cudaMemcpyAsync(h_ok, d_ok, n_ok, cudaMemcpyDeviceToHost, s));
    uint8_t* const h_sig = b->h_res + 64;
    uint8_t* const h_pk = h_sig + b->cap_sets;
    if (set_status) {
        LHB_CUDA(cudaMemcpyAsync(h_sig, b->d_status, b->n, cudaMemcpyDeviceToHost, s));
        LHB_CUDA(cudaMemcpyAsync(h_pk, b->d_pk_status, b->n, cudaMemcpyDeviceToHost, s));
    }
    if (b->n >= BLOCKING_WAIT_MIN_SETS && b->e_done) {
        // a long step: sleep on a blocking event instead of spinning in cudaStreamSynchronize — with one process per GPU
        // on a shared host (8 ranks + NCCL proxies under one cgroup CPU quota) eight spinning threads get throttled and
        // the next step's launches start late; the wake-up is noise against tens of milliseconds
        LHB_CUDA(cudaEventRecord(b->e_done, s));
        LHB_CUDA(cudaEventSynchronize(b->e_done));
    } else {
        LHB_CUDA(cudaStreamSynchronize(s));
    }
    memcpy(ok, h_ok, n_ok);
    // the two stages' codes for each set, the signature's first (the oracle checks the signature before the keys)
    if (set_status)
        for (uint32_t i = 0; i < b->n; i++) set_status[i] = h_sig[i] ? h_sig[i] : h_pk[i];
    return LHB200_OK;
}

int32_t lhb200_bls_batch_result(lhb200_bls_batch* b, void* stream, uint8_t* ok, uint8_t* set_status) {
    LHB_REQUIRE_READY();
    if (!b || !ok) return LHB200_EINVAL;
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    return fetch_results(b, s, b->d_ok, b->h_res, 1, ok, set_status);
}

// ---- segmented passes ------------------------------------------------------------------------------------------
int32_t lhb200_bls_batch_set_segments(lhb200_bls_batch* b, const uint32_t* batch_offsets, uint32_t n_batches) {
    LHB_REQUIRE_READY();
    const char* fn = "bls_batch_set_segments";
    if (!b || !batch_offsets || n_batches == 0) { set_error("%s: bad arguments", fn); return LHB200_EINVAL; }
    if (batch_offsets[0] != 0) { set_error("%s: offsets do not start at 0", fn); return LHB200_EINVAL; }
    uint32_t max_seg = 0;
    for (uint32_t k = 0; k < n_batches; k++) {
        if (batch_offsets[k + 1] <= batch_offsets[k]) { set_error("%s: empty or non-monotone segment", fn); return LHB200_EINVAL; }
        max_seg = std::max(max_seg, batch_offsets[k + 1] - batch_offsets[k]);
    }
    const uint32_t n = batch_offsets[n_batches], limit = pass_limit(g_cfg);
    if (n > b->cap_sets) { set_error("%s: more sets than the batch holds", fn); return LHB200_EINVAL; }
    if ((uint64_t)n + n_batches > limit) {
        set_error("%s: %u sets in %u segments exceed one pass (%u sets + segments)", fn, n, n_batches, limit);
        return LHB200_EINVAL;
    }
    if (!b->d_seg_off) {   // first segmented pass on this handle: buffers for the largest pass
#define ALLOC(p, bytes)                                                                                  \
    do {                                                                                                 \
        cudaError_t e = (p) ? cudaSuccess : cudaMalloc(reinterpret_cast<void**>(&(p)), (bytes));         \
        if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(" #p ")");                                 \
    } while (0)
        ALLOC(b->d_seg_sig, (size_t)limit * sizeof(G2Jac));
        ALLOC(b->d_seg_f, (size_t)limit * sizeof(Fp12));
        ALLOC(b->d_seg_gt, (size_t)limit * sizeof(Fp12));
        ALLOC(b->d_seg_ok, limit);
        if (!b->h_seg_ok) LHB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&b->h_seg_ok), limit, cudaHostAllocDefault));
        ALLOC(b->d_seg_off, (size_t)2 * (limit + 1) * 4);   // last: it marks the set as complete
#undef ALLOC
    }
    b->n = 0;   // inputs uploaded before do not carry the segments' grouping
    b->seg_h.assign(2 * (n_batches + 1), 0);
    memcpy(b->seg_h.data(), batch_offsets, (size_t)(n_batches + 1) * 4);
    b->max_seg = max_seg;
    b->n_seg = n_batches;
    return LHB200_OK;
}

int32_t lhb200_bls_batch_segment_result(lhb200_bls_batch* b, void* stream, uint8_t* ok, uint8_t* set_status) {
    LHB_REQUIRE_READY();
    if (!b || !ok || !b->n_seg_last) { set_error("bls_batch_segment_result: no segmented verify on this batch"); return LHB200_EINVAL; }
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    return fetch_results(b, s, b->d_seg_ok, b->h_seg_ok, b->n_seg_last, ok, set_status);
}

// Test hook: the value final_exp(product)^... of the last verify as 12 x 48-byte big-endian canonical Fp
// (order c0.c0.c0, c0.c0.c1, c0.c1.c0, ... c1.c2.c1).  It is the CUBE of the canonical GT element (pairing.cuh).
static void gt_to_bytes(const Fp12& f, uint8_t out576[576]) {
    const Fp* c = reinterpret_cast<const Fp*>(&f);
    // host-side conversion out of Montgomery form (plain integer arithmetic on 12 limbs, test hook only)
    for (int k = 0; k < 12; k++) {
        // t = c[k] * R^-1 mod p via 12 rounds of word-wise Montgomery reduction
        uint64_t t[13] = {0};
        for (int i = 0; i < 12; i++) t[i] = c[k].v[i];
        static const uint32_t P32[12] = {0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u,
                                         0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau};
        for (int i = 0; i < 12; i++) {
            const uint32_t m = (uint32_t)t[0] * 0xfffcfffdu;
            uint64_t carry = 0;
            for (int j = 0; j < 12; j++) {
                uint64_t v = t[j] + (uint64_t)m * P32[j] + carry;
                t[j] = v & 0xffffffffu;
                carry = v >> 32;
            }
            uint64_t top = t[12] + carry;
            for (int j = 0; j < 12; j++) t[j] = t[j + 1];
            t[11] = top & 0xffffffffu;
            t[12] = top >> 32;
        }
        // conditional subtract
        bool ge = t[12] != 0;
        if (!ge) {
            ge = true;
            for (int j = 11; j >= 0; j--) {
                if (t[j] != P32[j]) { ge = t[j] > P32[j]; break; }
            }
        }
        if (ge) {
            int64_t brw = 0;
            for (int j = 0; j < 12; j++) {
                int64_t v = (int64_t)t[j] - P32[j] - brw;
                brw = v < 0;
                t[j] = (uint64_t)(v & 0xffffffff);
            }
        }
        for (int j = 0; j < 12; j++) {
            uint8_t* q = out576 + 48 * k + 4 * (11 - j);
            q[0] = t[j] >> 24; q[1] = t[j] >> 16; q[2] = t[j] >> 8; q[3] = t[j];
        }
    }
}

int32_t lhb200_bls_batch_gt(lhb200_bls_batch* b, uint8_t out576[576]) {
    LHB_REQUIRE_READY();
    if (!b || !out576) return LHB200_EINVAL;
    Fp12 f;
    LHB_CUDA(cudaDeviceSynchronize());
    LHB_CUDA(cudaMemcpy(&f, b->d_gt, sizeof f, cudaMemcpyDeviceToHost));
    gt_to_bytes(f, out576);
    return LHB200_OK;
}

// Test hook: segment k's value of the last segmented verify, in the format of lhb200_bls_batch_gt.
int32_t lhb200_bls_batch_segment_gt(lhb200_bls_batch* b, uint32_t k, uint8_t out576[576]) {
    LHB_REQUIRE_READY();
    if (!b || !out576 || k >= b->n_seg_last) { set_error("bls_batch_segment_gt: no segment %u in the last verify", k); return LHB200_EINVAL; }
    Fp12 f;
    LHB_CUDA(cudaDeviceSynchronize());
    LHB_CUDA(cudaMemcpy(&f, b->d_seg_gt + k, sizeof f, cudaMemcpyDeviceToHost));
    gt_to_bytes(f, out576);
    return LHB200_OK;
}

uint64_t lhb200_bls_batch_launches(const lhb200_bls_batch* b) { return b ? b->launches_last : 0; }

// Test hook: the kernel choices of the last verify_enqueue (word layout in lhb200.h).
int32_t lhb200_bls_batch_plan(const lhb200_bls_batch* b, uint32_t* out, uint32_t n_words) {
    if (!b || (n_words && !out)) return LHB200_EINVAL;
    memcpy(out, b->plan, sizeof(uint32_t) * std::min<uint32_t>(n_words, LHB200_PLAN_WORDS));
    return LHB200_OK;
}

// Device time (ms, CUDA events on the launching stream) of the Miller kernel that ran in the last completed enqueue
// (k_miller_warp, k_miller_coop or k_miller_multi); negative if unavailable.  Call after the stream has been synchronised.
float lhb200_bls_batch_dominant_kernel_ms(const lhb200_bls_batch* b) {
    float ms = -1.f;
    if (!b || cudaEventElapsedTime(&ms, b->e_k0, b->e_k1) != cudaSuccess) { cudaGetLastError(); return -1.f; }
    return ms;
}

// bls::verify_signature_sets (crypto/bls/src/impls/blst.rs:37-119) on one pooled handle, alone.  Re-entrant: every call
// borrows a batch handle (device buffers, streams, events — no cudaMalloc on the steady path) from a pool and drives it
// on the handle's own stream, so concurrent calls overlap on the device instead of queueing behind one mutex.
static int32_t verify_alone(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks, const uint32_t* pk_offsets,
                            const uint64_t* rands, uint32_t n_sets, uint8_t* ok, uint8_t* set_status) {
    const uint64_t n_keys = pk_offsets[n_sets];
    lhb200_bls_batch* b = pool_acquire(n_sets, n_keys);
    if (!b) return LHB200_ENOMEM;
    int32_t rc = lhb200_bls_batch_upload_async(b, sigs, msgs, pks, pk_offsets, rands, n_sets, b->s_main);
    if (!rc) rc = lhb200_bls_batch_verify_enqueue(b, b->s_main);
    if (!rc) rc = lhb200_bls_batch_result(b, b->s_main, ok, set_status);
    cudaStreamSynchronize(b->s2);
    cudaStreamSynchronize(b->s3);
    pool_release(b);
    return rc;
}

// One segmented pass on a pooled handle: n sets (keys indexed from pk_offsets[0] == 0) in n_seg non-empty batches
// seg_off[0 .. n_seg] -> ok[n_seg] and, optionally, the n statuses.  rands NULL: drawn for the whole pass.
static int32_t verify_pass(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks, const uint32_t* pk_offsets,
                           const uint64_t* rands, uint32_t n, const uint32_t* seg_off, uint32_t n_seg, uint8_t* ok,
                           uint8_t* set_status) {
    lhb200_bls_batch* b = pool_acquire(n, pk_offsets[n]);
    if (!b) return LHB200_ENOMEM;
    int32_t rc = lhb200_bls_batch_set_segments(b, seg_off, n_seg);
    if (!rc) rc = lhb200_bls_batch_upload_async(b, sigs, msgs, pks, pk_offsets, rands, n, b->s_main);
    if (!rc) rc = lhb200_bls_batch_verify_enqueue(b, b->s_main);
    if (!rc) rc = lhb200_bls_batch_segment_result(b, b->s_main, ok, set_status);
    b->n_seg = 0;   // (left set by a failed upload)
    cudaStreamSynchronize(b->s2);
    cudaStreamSynchronize(b->s3);
    pool_release(b);
    return rc;
}

// The argument checks of the host uploads, made before a call is queued (so that its error is its own).
static int32_t check_sets(const char* fn, const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                          const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n) {
    if (n && (!sigs || !msgs || !pk_offsets)) { set_error("%s: bad arguments", fn); return LHB200_EINVAL; }
    for (uint32_t i = 0; i < n; i++)
        if (pk_offsets[i] > pk_offsets[i + 1]) { set_error("%s: offsets not monotone", fn); return LHB200_EINVAL; }
    if (n && pk_offsets[n] > pk_offsets[0] && !pks) { set_error("%s: no keys given", fn); return LHB200_EINVAL; }
    if (rands)
        for (uint32_t i = 0; i < n; i++)
            if (rands[i] == 0) { set_error("%s: zero random scalar", fn); return LHB200_EINVAL; }
    return LHB200_OK;
}

// ---- coalescing of concurrent plugin calls ----------------------------------------------------------------------
// Lighthouse calls verify_signature_sets from up to num_cpus blocking workers with <= 64-set gossip batches
// (beacon_processor/src/lib.rs:202-203,256).  Alone, such a batch is one wave of warps and a one-warp final
// exponentiation; concurrent calls are merged into segmented passes instead (leader / follower, no timer, no thread).
namespace {
constexpr uint32_t COALESCE_MAX_SETS = 64;   // calls above run alone: they are not what the gossip workers send
// Passes (lone calls included) on the device at once.  Measured on the H100 (DESIGN.md §2.7): with 2, 64 threads of
// 1-key gossip batches got 1.55x the batches/s of uncoalesced calls, but 8 and 16 threads lost a third (a lone call
// overlaps better with other lone calls than a queued call with a pass); with 8, 16 threads still lost 10-17 %.  With
// 16, up to 16 concurrent callers run exactly as before, and callers beyond them are merged.
constexpr uint32_t PASSES_IN_FLIGHT = 16;
struct Waiter {   // a queued call; its thread blocks in the call, so its buffers stay valid
    const uint8_t *sigs, *msgs, *pks;
    const uint32_t* pk_offsets;
    const uint64_t* rands;   // the caller's, or drawn by the caller
    uint32_t n;
    uint8_t *ok, *set_status;
    int32_t rc = LHB200_OK;
    std::string err;
    bool done = false;
};
std::mutex g_co_mu;
std::condition_variable g_co_cv;
uint32_t g_co_running = 0;   // passes in flight
std::deque<Waiter*> g_co_queue;

// The leader's work: the calls of `pass` as one segmented pass; every call gets its own verdict and statuses, or the
// pass's error.
void run_coalesced(const std::vector<Waiter*>& pass) {
    uint32_t n = 0;
    uint64_t n_keys = 0;
    for (const Waiter* w : pass) { n += w->n; n_keys += w->pk_offsets[w->n] - w->pk_offsets[0]; }
    std::vector<uint8_t> sigs((size_t)n * 96), msgs((size_t)n * 32), pks((size_t)n_keys * 96), st(n), ok(pass.size());
    std::vector<uint32_t> offs(n + 1), seg(pass.size() + 1);
    std::vector<uint64_t> rands(n);
    uint32_t lo = 0;
    uint64_t kb = 0;
    offs[0] = 0;
    for (size_t k = 0; k < pass.size(); k++) {
        const Waiter* w = pass[k];
        const uint32_t k0 = w->pk_offsets[0], kn = w->pk_offsets[w->n] - k0;
        seg[k] = lo;
        memcpy(&sigs[(size_t)96 * lo], w->sigs, (size_t)96 * w->n);
        memcpy(&msgs[(size_t)32 * lo], w->msgs, (size_t)32 * w->n);
        if (kn) memcpy(&pks[96 * kb], w->pks + (size_t)96 * k0, (size_t)96 * kn);
        memcpy(&rands[lo], w->rands, (size_t)8 * w->n);
        for (uint32_t i = 1; i <= w->n; i++) offs[lo + i] = (uint32_t)(kb + w->pk_offsets[i] - k0);
        lo += w->n;
        kb += kn;
    }
    seg[pass.size()] = n;
    const int32_t rc = verify_pass(sigs.data(), msgs.data(), pks.data(), offs.data(), rands.data(), n, seg.data(),
                                   (uint32_t)pass.size(), ok.data(), st.data());
    for (size_t k = 0; k < pass.size(); k++) {
        Waiter* w = pass[k];
        w->rc = rc;
        if (rc) { w->err = lhb200_last_error(); continue; }
        *w->ok = ok[k];
        if (w->set_status) memcpy(w->set_status, &st[seg[k]], w->n);
    }
}
}  // namespace

// bls::verify_signature_sets (crypto/bls/src/impls/blst.rs:37-119).  *ok = 1 iff every set verifies.
// n_sets == 0 -> *ok = 0 (blst.rs:42-44).  rands may be NULL (drawn internally, 64 nonzero bits each).
// set_status (optional, n bytes): per-set preparation status (0 = fine; see SetStatus in kernels.cuh).
int32_t lhb200_verify_signature_sets(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                     const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets, uint8_t* ok,
                                     uint8_t* set_status) {
    LHB_REQUIRE_READY();
    if (!ok) return LHB200_EINVAL;
    *ok = 0;
    if (n_sets == 0) return LHB200_OK;
    if (!pk_offsets) { set_error("verify_signature_sets: null offsets"); return LHB200_EINVAL; }
    if (n_sets > COALESCE_MAX_SETS) return verify_alone(sigs, msgs, pks, pk_offsets, rands, n_sets, ok, set_status);
    std::unique_lock<std::mutex> lk(g_co_mu);
    if (g_co_running < PASSES_IN_FLIGHT && g_co_queue.empty()) {   // a free slot: today's path, alone
        g_co_running++;
        lk.unlock();
        const int32_t rc = verify_alone(sigs, msgs, pks, pk_offsets, rands, n_sets, ok, set_status);
        lk.lock();
        g_co_running--;
        lk.unlock();
        g_co_cv.notify_all();
        return rc;
    }
    lk.unlock();
    // queue: this caller's own argument checks and scalars first
    if (int32_t rc = check_sets("verify_signature_sets", sigs, msgs, pks, pk_offsets, rands, n_sets)) return rc;
    std::vector<uint64_t> own_rands;
    if (!rands) {
        own_rands.resize(n_sets);
        if (!gen_rands(own_rands.data(), n_sets)) { set_error("verify_signature_sets: getrandom(2) failed"); return LHB200_ECUDA; }
        rands = own_rands.data();
    }
    Waiter me;
    me.sigs = sigs; me.msgs = msgs; me.pks = pks; me.pk_offsets = pk_offsets; me.rands = rands; me.n = n_sets;
    me.ok = ok; me.set_status = set_status;
    lk.lock();
    g_co_queue.push_back(&me);
    g_co_cv.wait(lk, [&] {   // (a leader may have taken this call already: the queue can be empty)
        return me.done || (!g_co_queue.empty() && g_co_queue.front() == &me && g_co_running < PASSES_IN_FLIGHT);
    });
    if (me.done) {   // a leader ran this call
        lk.unlock();
        if (me.rc) set_error("%s", me.err.c_str());
        return me.rc;
    }
    // leader: the waiting calls that fit one pass, in arrival order
    g_co_running++;
    std::vector<Waiter*> pass;
    uint32_t sets = 0;
    const uint32_t limit = pass_limit(g_cfg);
    while (!g_co_queue.empty() && sets + g_co_queue.front()->n + pass.size() + 1 <= limit) {
        pass.push_back(g_co_queue.front());
        sets += g_co_queue.front()->n;
        g_co_queue.pop_front();
    }
    lk.unlock();
    g_co_cv.notify_all();   // the next waiting call may lead the other slot
    if (pass.size() == 1) me.rc = verify_alone(sigs, msgs, pks, pk_offsets, rands, n_sets, ok, set_status);
    else run_coalesced(pass);
    lk.lock();
    for (Waiter* w : pass) w->done = true;
    g_co_running--;
    lk.unlock();
    g_co_cv.notify_all();
    if (me.rc && !me.err.empty()) set_error("%s", me.err.c_str());   // (a lone run set it on this thread already)
    return me.rc;
}

int32_t lhb200_verify_signature_set_batches(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                            const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets,
                                            const uint32_t* batch_offsets, uint32_t n_batches, uint8_t* ok,
                                            uint8_t* set_status) {
    LHB_REQUIRE_READY();
    const char* fn = "verify_signature_set_batches";
    if (n_batches == 0) return LHB200_OK;
    if (!ok || !batch_offsets || (n_sets && !pk_offsets)) { set_error("%s: bad arguments", fn); return LHB200_EINVAL; }
    if (batch_offsets[0] != 0 || batch_offsets[n_batches] != n_sets) {
        set_error("%s: batch offsets do not span the %u sets", fn, n_sets);
        return LHB200_EINVAL;
    }
    for (uint32_t k = 0; k < n_batches; k++)
        if (batch_offsets[k] > batch_offsets[k + 1]) { set_error("%s: batch offsets not monotone", fn); return LHB200_EINVAL; }
    if (int32_t rc = check_sets(fn, sigs, msgs, pks, pk_offsets, rands, n_sets)) return rc;
    const uint32_t limit = pass_limit(g_cfg);
    std::vector<uint32_t> offs, seg;
    for (uint32_t k = 0; k < n_batches;) {
        const uint32_t lo = batch_offsets[k];
        if (batch_offsets[k + 1] == lo) { ok[k++] = 0; continue; }   // an empty batch (blst.rs:42-44)
        if (batch_offsets[k + 1] - lo + 1 > limit) {                 // too large for a pass of its own
            const uint32_t n = batch_offsets[k + 1] - lo;
            offs.assign(pk_offsets + lo, pk_offsets + lo + n + 1);
            for (uint32_t& o : offs) o -= pk_offsets[lo];
            if (int32_t rc = verify_alone(sigs + (size_t)96 * lo, msgs + (size_t)32 * lo, pks + (size_t)96 * pk_offsets[lo],
                                          offs.data(), rands ? rands + lo : nullptr, n, ok + k,
                                          set_status ? set_status + lo : nullptr))
                return rc;
            k++;
            continue;
        }
        // the following non-empty batches while sets + batches fit one pass
        seg.assign(1, 0);
        uint32_t e = k;
        for (; e < n_batches && batch_offsets[e + 1] > batch_offsets[e] &&
               batch_offsets[e + 1] - lo + (e - k + 1) <= limit; e++)
            seg.push_back(batch_offsets[e + 1] - lo);
        const uint32_t n = batch_offsets[e] - lo;
        offs.assign(pk_offsets + lo, pk_offsets + lo + n + 1);
        for (uint32_t& o : offs) o -= pk_offsets[lo];
        if (int32_t rc = verify_pass(sigs + (size_t)96 * lo, msgs + (size_t)32 * lo, pks + (size_t)96 * pk_offsets[lo],
                                     offs.data(), rands ? rands + lo : nullptr, n, seg.data(), e - k, ok + k,
                                     set_status ? set_status + lo : nullptr))
            return rc;
        k = e;
    }
    return LHB200_OK;
}

// verify_signature_sets over the ranks of the library's communicator: every rank passes ITS shard of the sets (possibly
// empty: an empty shard contributes `true`), runs the batch check on it with its own blinding scalars and final
// exponentiation, and the verdicts are combined by one ncclAllReduce(min) on the device (SURVEY.md §8e option (a)).
// *ok is the verdict of the WHOLE batch on every rank.  Without a communicator this is lhb200_verify_signature_sets
// (except that n_sets == 0 yields *ok = 1: "this shard has nothing to object to").
int32_t lhb200_verify_signature_sets_collective(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                                const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets,
                                                uint8_t* ok) {
    LHB_REQUIRE_READY();
    if (!ok) return LHB200_EINVAL;
    *ok = 0;
    if (n_sets && !pk_offsets) return LHB200_EINVAL;
    const uint64_t n_keys = n_sets ? pk_offsets[n_sets] : 0;
    lhb200_bls_batch* b = pool_acquire(std::max<uint32_t>(n_sets, 1), n_keys);
    if (!b) return LHB200_ENOMEM;
    int32_t rc = LHB200_OK;
    if (n_sets) {
        rc = lhb200_bls_batch_upload_async(b, sigs, msgs, pks, pk_offsets, rands, n_sets, b->s_main);
        if (!rc) rc = lhb200_bls_batch_verify_enqueue(b, b->s_main);
    } else {
        const uint8_t one = 1;
        cudaError_t e = cudaMemcpyAsync(b->d_ok, &one, 1, cudaMemcpyHostToDevice, b->s_main);
        if (e == cudaSuccess) e = cudaStreamSynchronize(b->s_main);   // `one` is a stack variable
        if (e != cudaSuccess) rc = cuda_fail(e, "empty shard verdict");
        b->n = 0;
    }
    if (!rc) rc = comm_allreduce_min_u8(b->d_ok, 1, b->s_main);
    if (!rc) rc = lhb200_bls_batch_result(b, b->s_main, ok, nullptr);
    cudaStreamSynchronize(b->s2);
    cudaStreamSynchronize(b->s3);
    pool_release(b);
    return rc;
}

// TSecretKey::public_key (blst.rs:282-298): n big-endian 32-byte scalars -> compressed (48 B) and/or
// uncompressed (96 B) public keys.  Either output may be NULL.
int32_t lhb200_sk_to_pk(const uint8_t* sk32, uint32_t n, uint8_t* pk48, uint8_t* pk96) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!sk32 || (!pk48 && !pk96)) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch((size_t)n * (32 + 48 + 96) + 1024));
    if (!d) return LHB200_ENOMEM;
    uint8_t *d48 = d + (size_t)n * 32, *d96 = d48 + (size_t)n * 48;
    LHB_CUDA(cudaMemcpyAsync(d, sk32, (size_t)n * 32, cudaMemcpyHostToDevice, c.stream));
    k_sk_to_pk<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, pk48 ? d48 : nullptr, pk96 ? d96 : nullptr);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    if (pk48) LHB_CUDA(cudaMemcpyAsync(pk48, d48, (size_t)n * 48, cudaMemcpyDeviceToHost, c.stream));
    if (pk96) LHB_CUDA(cudaMemcpyAsync(pk96, d96, (size_t)n * 96, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

// TSecretKey::sign (blst.rs:282-298 / generic_secret_key.rs): sig_i = sk_i * H(msg_i), compressed 96 B.
int32_t lhb200_sign(const uint8_t* sk32, const uint8_t* msg32, uint32_t n, uint8_t* sig96) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!sk32 || !msg32 || !sig96) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch((size_t)n * (32 + 32 + 96) + 1024));
    if (!d) return LHB200_ENOMEM;
    uint8_t *dm = d + (size_t)n * 32, *ds = dm + (size_t)n * 32;
    LHB_CUDA(cudaMemcpyAsync(d, sk32, (size_t)n * 32, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemcpyAsync(dm, msg32, (size_t)n * 32, cudaMemcpyHostToDevice, c.stream));
    k_sign<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, dm, n, ds);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(sig96, ds, (size_t)n * 96, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

// PublicKey::deserialize + key_validate for n compressed keys (blst.rs:130-140; the batch form of
// validator_pubkey_cache.rs:116-118).  status[i]: 0 ok, 1 infinity (rejected, generic_public_key.rs:87-88),
// 2 bad encoding / not on curve, 3 not in the r-order subgroup.  pk96[i] is zeroed unless status is 0.
int32_t lhb200_g1_decompress_validate(const uint8_t* pk48, uint32_t n, uint8_t* pk96, uint8_t* status) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!pk48 || !pk96 || !status) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch((size_t)n * (48 + 96 + 1) + 1024));
    if (!d) return LHB200_ENOMEM;
    uint8_t *d96 = d + (size_t)n * 48, *dst = d96 + (size_t)n * 96;
    LHB_CUDA(cudaMemcpyAsync(d, pk48, (size_t)n * 48, cudaMemcpyHostToDevice, c.stream));
    k_g1_decompress_validate<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, d96, dst);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(pk96, d96, (size_t)n * 96, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(status, dst, n, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

// Signature::deserialize for n compressed signatures (blst.rs:192-194): 192-byte affine out
// (x.c1 | x.c0 | y.c1 | y.c0), status[i]: 0 ok, 1 infinity, 2 bad encoding / not on curve.  No subgroup check.
int32_t lhb200_g2_decompress(const uint8_t* sig96, uint32_t n, uint8_t* out192, uint8_t* status) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!sig96 || !out192 || !status) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch((size_t)n * (96 + 192 + 1) + 1024));
    if (!d) return LHB200_ENOMEM;
    uint8_t *do_ = d + (size_t)n * 96, *dst = do_ + (size_t)n * 192;
    LHB_CUDA(cudaMemcpyAsync(d, sig96, (size_t)n * 96, cudaMemcpyHostToDevice, c.stream));
    k_g2_decompress<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, do_, dst);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(out192, do_, (size_t)n * 192, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(status, dst, n, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}


// ---- aggregation surface of a crypto/bls backend --------------------------------------------------------------
// TAggregateSignature::add_assign / add_assign_aggregate (blst.rs:230-237) and AggregateSignature aggregation in
// general: out = sum of n compressed signatures.  No subgroup check (blst.rs:231: "signature has already been subgroup
// checked"); infinity encodings are the identity; n == 0 gives the infinity signature.  LHB200_EDECODE if any encoding
// is malformed.
int32_t lhb200_g2_aggregate(const uint8_t* sigs96, uint32_t n, uint8_t out96[96]) {
    LHB_REQUIRE_READY();
    if (!out96 || (n && !sigs96)) return LHB200_EINVAL;
    if (n == 0) { memset(out96, 0, 96); out96[0] = 0xc0; return LHB200_OK; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const uint64_t n1 = cdiv(n, REDUCE_CHUNK) + 1;
    const size_t b_in = ((size_t)n * 96 + 255) / 256 * 256, b_pts = (size_t)n * sizeof(G2Jac), b_t = (size_t)n1 * sizeof(G2Jac);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(b_in + b_pts + 2 * b_t + 512));
    if (!d) return LHB200_ENOMEM;
    G2Jac* pts = reinterpret_cast<G2Jac*>(d + b_in);
    G2Jac* tmp[2] = {reinterpret_cast<G2Jac*>(d + b_in + b_pts), reinterpret_cast<G2Jac*>(d + b_in + b_pts + b_t)};
    uint8_t* d_out = d + b_in + b_pts + 2 * b_t;
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(d_out + 128);
    LHB_CUDA(cudaMemcpyAsync(d, sigs96, (size_t)n * 96, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemsetAsync(d_bad, 0, 4, c.stream));
    k_g2_load_points<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, pts, d_bad);
    const uint32_t levels = tree_levels(n, REDUCE_CHUNK, 1);
    const G2Jac* sum = reduce_tree<G2Jac>(pts, n, REDUCE_CHUNK, levels, tmp, [&](const G2Jac* in, uint32_t m, uint32_t mo, G2Jac* out) {
        k_g2_reduce<<<cdiv(mo, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(in, m, REDUCE_CHUNK, out);
    });
    k_g2_store_point<<<1, 32, 0, c.stream>>>(sum, d_out);
    count_launch(2 + levels);
    LHB_CUDA(cudaGetLastError());
    uint8_t h[96];
    uint32_t bad = 0;
    LHB_CUDA(cudaMemcpyAsync(h, d_out, 96, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    if (bad) { set_error("g2_aggregate: %u malformed signature encodings", bad); return LHB200_EDECODE; }
    memcpy(out96, h, 96);
    return LHB200_OK;
}

// TAggregatePublicKey::aggregate (blst.rs:178-184): sum of n uncompressed keys ("already checked for subgroup and
// infinity"), both serialisations out (either may be NULL).  n == 0 -> LHB200_EINVAL (blst: AGGR_TYPE_MISMATCH).
// Malformed / off-curve key -> LHB200_EDECODE.
int32_t lhb200_g1_aggregate(const uint8_t* pks96, uint32_t n, uint8_t* out48, uint8_t* out96) {
    LHB_REQUIRE_READY();
    if (!pks96 || n == 0 || (!out48 && !out96)) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const uint64_t n1 = cdiv(n, REDUCE_CHUNK) + 1;
    const size_t b_in = ((size_t)n * 96 + 255) / 256 * 256, b_pts = (size_t)n * sizeof(G1Jac), b_t = (size_t)n1 * sizeof(G1Jac);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(b_in + b_pts + 2 * b_t + 512));
    if (!d) return LHB200_ENOMEM;
    G1Jac* pts = reinterpret_cast<G1Jac*>(d + b_in);
    G1Jac* tmp[2] = {reinterpret_cast<G1Jac*>(d + b_in + b_pts), reinterpret_cast<G1Jac*>(d + b_in + b_pts + b_t)};
    uint8_t* d_out = d + b_in + b_pts + 2 * b_t;
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(d_out + 256);
    LHB_CUDA(cudaMemcpyAsync(d, pks96, (size_t)n * 96, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemsetAsync(d_bad, 0, 4, c.stream));
    k_g1_load_points<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, pts, nullptr, nullptr, d_bad);
    const uint32_t levels = tree_levels(n, REDUCE_CHUNK, 1);
    const G1Jac* sum = reduce_tree<G1Jac>(pts, n, REDUCE_CHUNK, levels, tmp, [&](const G1Jac* in, uint32_t m, uint32_t mo, G1Jac* out) {
        k_g1_reduce<<<cdiv(mo, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(in, m, REDUCE_CHUNK, out);
    });
    k_g1_store_point<<<1, 32, 0, c.stream>>>(sum, d_out, d_out + 64);
    count_launch(2 + levels);
    LHB_CUDA(cudaGetLastError());
    uint8_t h[160];
    uint32_t bad = 0;
    LHB_CUDA(cudaMemcpyAsync(h, d_out, 160, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    if (bad) { set_error("g1_aggregate: %u malformed or off-curve keys", bad); return LHB200_EDECODE; }
    if (out48) memcpy(out48, h, 48);
    if (out96) memcpy(out96, h + 64, 96);
    return LHB200_OK;
}

// TPublicKey::deserialize_uncompressed (blst.rs:142-150), batch form: encoding and on-curve checks, NO subgroup check
// (blst's P1 deserialize does none).  status[i]: 0 ok, 1 infinity, 2 bad encoding / not on the curve.  pk48 (optional):
// the compressed form of every accepted key (zeros otherwise).
int32_t lhb200_g1_deserialize_uncompressed(const uint8_t* pks96, uint32_t n, uint8_t* pk48, uint8_t* status) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!pks96 || !status) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const size_t b_in = ((size_t)n * 96 + 255) / 256 * 256, b_48 = ((size_t)n * 48 + 255) / 256 * 256;
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(b_in + b_48 + n + 512));
    if (!d) return LHB200_ENOMEM;
    uint8_t *d48 = d + b_in, *dst = d48 + b_48;
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(dst + (n + 255) / 256 * 256);
    LHB_CUDA(cudaMemcpyAsync(d, pks96, (size_t)n * 96, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemsetAsync(d_bad, 0, 4, c.stream));
    k_g1_load_points<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, c.stream>>>(d, n, nullptr, pk48 ? d48 : nullptr, dst, d_bad);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    if (pk48) LHB_CUDA(cudaMemcpyAsync(pk48, d48, (size_t)n * 48, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(status, dst, n, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

// TAggregateSignature::aggregate_verify (blst.rs:263-273; generic_aggregate_signature.rs:213-222):
// e(g1, sig) == prod_i e(pk_i, H(m_i)) with the signature subgroup-checked.  n == 0 -> *ok = 0.
// Runs on the batch pipeline: set 0 carries `sig`, the other sets the infinity signature, all blinding scalars are 1,
// so prod_i e(pk_i, H(m_i)) * e(-g1, sig) == 1 is exactly the check.
int32_t lhb200_aggregate_verify(const uint8_t sig96[96], const uint8_t* msgs, const uint8_t* pks96, uint32_t n, uint8_t* ok) {
    LHB_REQUIRE_READY();
    if (!ok) return LHB200_EINVAL;
    *ok = 0;
    if (n == 0) return LHB200_OK;
    if (!sig96 || !msgs || !pks96) return LHB200_EINVAL;
    std::vector<uint8_t> sigs((size_t)n * 96, 0);
    std::vector<uint32_t> offs(n + 1);
    std::vector<uint64_t> ones(n, 1);
    memcpy(sigs.data(), sig96, 96);
    for (uint32_t i = 1; i < n; i++) sigs[(size_t)i * 96] = 0xc0;
    for (uint32_t i = 0; i <= n; i++) offs[i] = i;
    return lhb200_verify_signature_sets(sigs.data(), msgs, pks96, offs.data(), ones.data(), n, ok, nullptr);
}

// Test hook: run one pipeline stage on a single device thread (op codes in bls/debug.cuh).
int32_t lhb200_debug_bls(int32_t op, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t out_len, int32_t* rc) {
    LHB_REQUIRE_READY();
    if (!in || !out || !rc) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch((size_t)in_len + out_len + 1024));
    if (!d) return LHB200_ENOMEM;
    uint8_t* d_out = d + ((in_len + 255) / 256) * 256;
    int32_t* d_rc = reinterpret_cast<int32_t*>(d_out + ((out_len + 255) / 256) * 256);
    LHB_CUDA(cudaMemcpyAsync(d, in, in_len, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemsetAsync(d_out, 0, out_len, c.stream));
    k_debug_bls<<<1, 32, 0, c.stream>>>(op, d, d_out, d_rc);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(out, d_out, out_len, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaMemcpyAsync(rc, d_rc, 4, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

}  // extern "C"
