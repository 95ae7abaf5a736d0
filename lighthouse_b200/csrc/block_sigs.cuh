// block_sigs.cuh — the signature sets of SignedBeaconBlocks on the device (lhb200_block_signatures_verify, sm_90a).
//
//   k_block_set_roots ........... one thread per set the host described: the object root (a caller's block root, an
//                                 epoch, a BeaconBlockHeader, an AttestationData, a VoluntaryExit, a Consolidation or a
//                                 BlsToExecutionChange read from the staged blocks), the fork-data root of the set's
//                                 domain and the signing root (signature_sets.rs, SigningData)
//   k_sync_committee_resolve .... one pass over the resident validator records against a shared-memory table of the
//                                 512 current_sync_committee pubkeys: the smallest validator index holding each member's
//                                 key (the pubkey cache lookup of block_verification.rs:2127-2132)
// Attestations go through k_attestation_index_count / k_attestation_index_write (attest.cuh).
#pragma once
#include "attest.cuh"

namespace lhb200 {

// What a set signs: hash_tree_root of the object at `off` in the staged blob (or of `epoch`), and
// compute_domain(domain, version, genesis_validators_root) with the version the host chose
enum : uint32_t { BSO_ROOT = 0, BSO_EPOCH, BSO_HEADER, BSO_ATT_DATA, BSO_EXIT, BSO_CONSOLIDATION, BSO_BLS_CHANGE };
struct BlockSetDesc {
    uint64_t off;        // byte offset of the object in the staged blob (BSO_EPOCH: unused)
    uint64_t epoch;      // BSO_EPOCH: the signed epoch
    uint32_t object;     // BSO_*
    uint32_t domain;     // the domain type as the first big-endian word of the domain (type 1 -> 0x01000000)
    uint32_t version;    // the fork version as a big-endian word
    uint32_t pad;
};
struct BlockRootParams {
    const uint8_t* blob;
    const BlockSetDesc* desc;
    uint32_t n;
    uint32_t gvr[8];
    uint8_t* roots;      // n x 32 signing roots
};

constexpr int BLOCK_ROOT_THREADS = 128;
__global__ void __launch_bounds__(BLOCK_ROOT_THREADS) k_block_set_roots(const __grid_constant__ BlockRootParams p) {
    const uint32_t i = blockIdx.x * BLOCK_ROOT_THREADS + threadIdx.x;
    if (i >= p.n) return;
    const BlockSetDesc ds = p.desc[i];
    const uint8_t* o = p.blob + ds.off;
    uint32_t h[8], a[8], b[8];
    switch (ds.object) {
    case BSO_ROOT: h256_chunk(o, h); break;
    case BSO_EPOCH:
#pragma unroll
        for (int k = 0; k < 8; k++) h[k] = 0;
        h[0] = bswap32((uint32_t)ds.epoch);
        h[1] = bswap32((uint32_t)(ds.epoch >> 32));
        break;
    case BSO_HEADER:   // BeaconBlockHeader {slot, proposer_index, parent_root, state_root, body_root}: 8 leaves
        u64_chunk(o, a); u64_chunk(o + 8, b); hash_pair_inl(a, b, h);
        h256_chunk(o + 16, a); h256_chunk(o + 48, b); hash_pair_inl(a, b, a);
        hash_pair_inl(h, a, h);
        h256_chunk(o + 80, a); hash_pair_inl(a, g_zero_words[0], a);
        hash_pair_inl(a, g_zero_words[1], a);
        hash_pair_inl(h, a, h);
        break;
    case BSO_ATT_DATA: attestation_data_root_words(o, h); break;
    case BSO_EXIT:     // VoluntaryExit {epoch, validator_index}
        u64_chunk(o, a); u64_chunk(o + 8, b); hash_pair_inl(a, b, h);
        break;
    case BSO_CONSOLIDATION:   // Consolidation {source_index, target_index, epoch}: 4 leaves
        u64_chunk(o, a); u64_chunk(o + 8, b); hash_pair_inl(a, b, h);
        u64_chunk(o + 16, a); hash_pair_inl(a, g_zero_words[0], a);
        hash_pair_inl(h, a, h);
        break;
    default:           // BlsToExecutionChange {validator_index, from_bls_pubkey: 48 B, to_execution_address: 20 B}
        h256_chunk(o + 8, a);
#pragma unroll
        for (int k = 0; k < 8; k++) b[k] = k < 4 ? be_word(o + 40 + 4 * k) : 0;
        hash_pair_inl(a, b, b);                                 // the pubkey's root
        u64_chunk(o, a); hash_pair_inl(a, b, h);
#pragma unroll
        for (int k = 0; k < 8; k++) a[k] = k < 5 ? be_word(o + 56 + 4 * k) : 0;
        hash_pair_inl(a, g_zero_words[0], a);
        hash_pair_inl(h, a, h);
    }
    // domain = type || hash_tree_root(ForkData { version, genesis_validators_root })[0 .. 28)
    uint32_t d[8];
#pragma unroll
    for (int k = 1; k < 8; k++) d[k] = 0;
    d[0] = ds.version;
    hash_pair_inl(d, p.gvr, d);
#pragma unroll
    for (int k = 7; k > 0; k--) d[k] = d[k - 1];
    d[0] = ds.domain;
    hash_pair_inl(h, d, h);
    store_chunk(p.roots + 32ull * i, h);
}

constexpr uint32_t SYNC_MEMBERS = 512, SYNC_SLOTS = 1024;   // open addressing at load 1/2
constexpr int SYNC_RESOLVE_THREADS = 256;
__device__ __forceinline__ uint64_t pk_key8(const uint8_t* pk) {
    uint64_t v = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) v |= (uint64_t)pk[k] << (8 * k);
    return v;
}
__device__ __forceinline__ uint32_t pk_slot(uint64_t key) { return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 54); }

// out[m] = the smallest index v < n whose record's pubkey equals member m's (atomicMin; the caller fills out with
// 0xFF bytes first, so UINT32_MAX stays for a key no record holds).  Members with one key take separate slots.
__global__ void __launch_bounds__(SYNC_RESOLVE_THREADS) k_sync_committee_resolve(const uint8_t* __restrict__ vals,
                                                                                uint64_t n,
                                                                                const uint8_t* __restrict__ committee,
                                                                                uint32_t* __restrict__ out) {
    __shared__ uint64_t s_key[SYNC_SLOTS];
    __shared__ uint32_t s_member[SYNC_SLOTS];
    for (uint32_t k = threadIdx.x; k < SYNC_SLOTS; k += SYNC_RESOLVE_THREADS) s_member[k] = UINT32_MAX;
    __syncthreads();
    for (uint32_t m = threadIdx.x; m < SYNC_MEMBERS; m += SYNC_RESOLVE_THREADS) {
        const uint64_t key = pk_key8(committee + 48 * m);
        uint32_t h = pk_slot(key);
        while (atomicCAS(&s_member[h], UINT32_MAX, m) != UINT32_MAX) h = (h + 1) & (SYNC_SLOTS - 1);
        s_key[h] = key;
    }
    __syncthreads();
    for (uint64_t v = blockIdx.x * (uint64_t)SYNC_RESOLVE_THREADS + threadIdx.x; v < n;
         v += (uint64_t)gridDim.x * SYNC_RESOLVE_THREADS) {
        const uint8_t* pk = vals + 121 * v;
        const uint64_t key = pk_key8(pk);
        for (uint32_t h = pk_slot(key), m; (m = s_member[h]) != UINT32_MAX; h = (h + 1) & (SYNC_SLOTS - 1)) {
            if (s_key[h] != key) continue;
            const uint8_t* c = committee + 48 * m;
            bool eq = true;
            for (int k = 8; k < 48 && eq; k++) eq = c[k] == pk[k];
            if (eq) atomicMin(&out[m], (uint32_t)v);
        }
    }
}

}  // namespace lhb200
