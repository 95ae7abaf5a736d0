// attest.cuh — Attestation indexing and signing roots on the device (lhb200_attestations_verify, sm_90a).
//
//   k_attestation_index_count ... one warp per Attestation: framing, committee lookup in a resident committee cache,
//                                 set-bit count, the unknown-validator check, the AttestationData root and the signing
//                                 root (get_attesting_indices.rs, signature_sets.rs:271-332)
//   k_attestation_index_write ... one CTA per Attestation: the attesting indices in committee order into the BLS batch's
//                                 key-index buffer and, on request, into the indexed output (sorted in shared memory
//                                 before Electra; staged for one segmented sort in Electra)
#pragma once
#include "merkle.cuh"

namespace lhb200 {

// Attestation SSZ: {aggregation_bits offset (4 B), data: AttestationData (128 B at 4), signature (96 B at 132)} and,
// from Electra, committee_bits: Bitvector[64] (8 B at 228); then the bitlist bytes with their delimiter.
constexpr uint32_t ATT_DATA = 4, ATT_SIG = 132, ATT_COMMITTEE_BITS = 228;
constexpr uint32_t ATT_FIXED = 228, ATT_FIXED_ELECTRA = 236;
constexpr uint32_t ATT_MAX_BITS = 2048, ATT_MAX_BITS_ELECTRA = 131072;   // MaxValidatorsPerCommittee, MaxValidatorsPerSlot
constexpr uint32_t ATT_MAX_CACHES = 3, ATT_MAX_COMMITTEES = 64;
// Per-attestation status (lhb200.h): 0 fine, then the indexing errors in the order the reference meets them
enum : uint8_t {
    ATT_OK = 0, ATT_MALFORMED = 10, ATT_NO_CACHE = 11, ATT_NO_COMMITTEE = 12, ATT_BITFIELD_LENGTH = 13,
    ATT_UNKNOWN_VALIDATOR = 14
};

struct AttCache {
    const uint64_t* shuffling;   // n_active shuffled active indices
    uint64_t epoch;
    uint32_t n_active, committees_per_slot;
};
struct AttParams {
    const uint8_t* ssz;          // the records; record i is [offs[i] - offs[0], offs[i + 1] - offs[0])
    const uint64_t* offs;        // n + 1
    uint32_t n, electra, n_caches;
    AttCache cache[ATT_MAX_CACHES];
    uint64_t table_len, fork_epoch;
    uint32_t version[2];         // the previous / current fork version, as a big-endian word
    uint32_t gvr[8];             // genesis_validators_root, in word form
    uint8_t* roots;              // n x 32 signing roots, then the n u32 counts, then the n status bytes
    uint32_t* counts;
    uint8_t* status;
};

__device__ __forceinline__ uint64_t att_u64(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) v = (v << 8) | p[k];
    return v;
}

// hash_tree_root of the 128-byte AttestationData at d {slot, index, beacon_block_root, source, target}: 8 leaves (each
// checkpoint a 2-leaf container), 7 hashes, the compressions inlined (k_pending_attestation_roots hashes the same
// container out of line, inside its record)
__device__ __forceinline__ void attestation_data_root_words(const uint8_t* d, uint32_t t[8]) {
    uint32_t a[8], b[8];
    u64_chunk(d, a); u64_chunk(d + 8, b); hash_pair_inl(a, b, t);                    // H(slot, index)
    u64_chunk(d + 48, a); h256_chunk(d + 56, b); hash_pair_inl(a, b, b);             // source
    h256_chunk(d + 16, a); hash_pair_inl(a, b, a);                                   // H(beacon_block_root, source)
    hash_pair_inl(t, a, t);
    u64_chunk(d + 88, a); h256_chunk(d + 96, b); hash_pair_inl(a, b, a);             // target
    hash_pair_inl(a, g_zero_words[0], a);
    hash_pair_inl(a, g_zero_words[1], a);
    hash_pair_inl(t, a, t);
}

// Frames record i: its fixed part, the offset that must point right behind it, and a bitlist of 1 to max bits with its
// delimiter.  Only the host-checked offsets decide where a read goes; the record's own bytes never do.
__device__ __forceinline__ bool att_frame(const AttParams& p, uint32_t i, const uint8_t*& r, uint32_t& nb,
                                          uint32_t& n_bits) {
    const uint32_t fixed = p.electra ? ATT_FIXED_ELECTRA : ATT_FIXED;
    const uint32_t max_bits = p.electra ? ATT_MAX_BITS_ELECTRA : ATT_MAX_BITS;
    const uint64_t lo = p.offs[i] - p.offs[0], len = p.offs[i + 1] - p.offs[i];
    if (len < fixed + 1 || len > fixed + max_bits / 8 + 1) return false;
    r = p.ssz + lo;
    if (le_u32(r) != fixed) return false;
    nb = (uint32_t)len - fixed;
    const uint32_t last = r[fixed + nb - 1];
    if (last == 0) return false;
    n_bits = 8 * (nb - 1) + 31 - __clz(last);
    return n_bits <= max_bits;
}

// The committees of a framed record (get_attesting_indices.rs): the cache of data.slot's epoch (ci), then the
// committees in aggregation-bit order.  seg_bit[k] is committee k's first bit, seg_start[k] its first position in the
// shuffling, seg_bit[n_seg] the bits they cover.  -> ATT_OK or the first indexing error the reference reports.
__device__ __forceinline__ uint32_t att_committees(const AttParams& p, const uint8_t* r, uint32_t n_bits, uint32_t& ci,
                                                uint32_t* seg_bit, uint32_t* seg_start, uint32_t& n_seg) {
    const uint64_t slot = att_u64(r + ATT_DATA), epoch = slot / 32;
    ci = ATT_MAX_CACHES;
    for (uint32_t k = 0; k < p.n_caches; k++)
        if (p.cache[k].epoch == epoch) ci = k;
    if (ci == ATT_MAX_CACHES) { ci = 0; return ATT_NO_CACHE; }
    const AttCache& c = p.cache[ci];
    const uint64_t cps = c.committees_per_slot, count = cps * 32, n = c.n_active;
    // committee_cache.rs:313-330 (compute_committee_range_in_epoch)
    auto range = [&](uint64_t index, uint32_t& start, uint32_t& len) {
        const uint64_t k = (slot % 32) * cps + index, s = n * k / count;
        start = (uint32_t)s;
        len = (uint32_t)(n * (k + 1) / count - s);
    };
    n_seg = 0;
    uint32_t total = 0;
    if (!p.electra) {
        const uint64_t index = att_u64(r + ATT_DATA + 8);
        if (index >= cps) return ATT_NO_COMMITTEE;
        uint32_t start, len;
        range(index, start, len);
        seg_bit[0] = 0;
        seg_start[0] = start;
        n_seg = 1;
        total = len;
    } else {
        for (uint64_t bits = att_u64(r + ATT_COMMITTEE_BITS); bits; bits &= bits - 1) {
            const uint64_t index = __ffsll((long long)bits) - 1;
            if (index >= cps) return ATT_NO_COMMITTEE;
            uint32_t start, len;
            range(index, start, len);
            seg_bit[n_seg] = total;
            seg_start[n_seg] = start;
            n_seg++;
            total += len;
        }
    }
    seg_bit[n_seg] = total;
    return total == n_bits ? ATT_OK : ATT_BITFIELD_LENGTH;
}

// Position in the shuffling of aggregation bit q: committee = the last one whose first bit is <= q
__device__ __forceinline__ uint32_t att_position(const uint32_t* seg_bit, const uint32_t* seg_start, uint32_t n_seg,
                                                 uint32_t q) {
    uint32_t lo = 0, hi = n_seg;   // seg_bit[lo] <= q < seg_bit[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (seg_bit[mid] <= q) lo = mid;
        else hi = mid;
    }
    return seg_start[lo] + q - seg_bit[lo];
}

constexpr int ATT_COUNT_WARPS = 4;
__global__ void __launch_bounds__(32 * ATT_COUNT_WARPS) k_attestation_index_count(const __grid_constant__ AttParams p) {
    __shared__ uint32_t s_bit[ATT_COUNT_WARPS][ATT_MAX_COMMITTEES + 1], s_start[ATT_COUNT_WARPS][ATT_MAX_COMMITTEES];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, i = blockIdx.x * ATT_COUNT_WARPS + w;
    if (i >= p.n) return;   // the whole warp
    const uint32_t fixed = p.electra ? ATT_FIXED_ELECTRA : ATT_FIXED;
    const uint8_t* r = nullptr;
    uint32_t nb = 0, n_bits = 0, ci = 0, n_seg = 0;
    uint32_t st = att_frame(p, i, r, nb, n_bits) ? ATT_OK : ATT_MALFORMED;
    if (st == ATT_OK && lane == 0) st = att_committees(p, r, n_bits, ci, s_bit[w], s_start[w], n_seg);
    st = __shfl_sync(0xffffffffu, st, 0);
    ci = __shfl_sync(0xffffffffu, ci, 0);
    n_seg = __shfl_sync(0xffffffffu, n_seg, 0);
    __syncwarp();
    uint32_t cnt = 0;
    if (st == ATT_OK) {
        // set bits, and whether one names a validator beyond the pubkey table (ValidatorUnknown)
        const uint64_t* sh = p.cache[ci].shuffling;
        bool unknown = false;
        for (uint32_t b = lane; b < nb; b += 32) {
            uint32_t v = r[fixed + b];
            if (b + 1 == nb) v &= ~(0x80000000u >> __clz(v));   // the delimiter
            cnt += __popc(v);
            for (; v; v &= v - 1) {
                const uint32_t q = 8 * b + __ffs(v) - 1;
                unknown |= sh[att_position(s_bit[w], s_start[w], n_seg, q)] >= p.table_len;
            }
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (__any_sync(0xffffffffu, unknown)) st = ATT_UNKNOWN_VALIDATOR;
    }
    if (lane == 0) {
        uint32_t h[8];
        if (st != ATT_MALFORMED) {
            // signing_root = H(hash_tree_root(data) || domain), domain = compute_domain(DOMAIN_BEACON_ATTESTER,
            // version of the fork at target.epoch, gvr) = 01 00 00 00 || fork_data_root[0 .. 28)
            const uint64_t target_epoch = att_u64(r + ATT_DATA + 88);
            uint32_t d[8];
#pragma unroll
            for (int k = 1; k < 8; k++) d[k] = 0;
            d[0] = p.version[target_epoch < p.fork_epoch ? 0 : 1];
            hash_pair_inl(d, p.gvr, d);   // hash_tree_root(ForkData { version, genesis_validators_root })
#pragma unroll
            for (int k = 7; k > 0; k--) d[k] = d[k - 1];
            d[0] = 0x01000000u;       // DOMAIN_BEACON_ATTESTER, little-endian u32
            attestation_data_root_words(r + ATT_DATA, h);
            hash_pair_inl(h, d, h);
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) h[k] = 0;
        }
        store_chunk(p.roots + 32ull * i, h);
        p.counts[i] = cnt;
        p.status[i] = (uint8_t)st;
    }
}

constexpr int ATT_WRITE_THREADS = 256;
constexpr uint32_t ATT_SORT_MAX = ATT_MAX_BITS;   // the shared-memory sort takes a pre-Electra committee
struct AttWrite {
    const uint32_t* key_off;     // n: first slot of the attestation's keys in `keys`; UINT32_MAX: not in the batch
    uint32_t* keys;              // the BLS batch's key-index buffer
    const uint64_t* out_off;     // n + 1: CSR of the indexed output (nullptr: no output)
    uint64_t* out;               // sorted indices (pre-Electra), or unsorted for the segmented sort (Electra)
};

__global__ void __launch_bounds__(ATT_WRITE_THREADS) k_attestation_index_write(const __grid_constant__ AttParams p,
                                                                               const __grid_constant__ AttWrite wr) {
    __shared__ uint32_t s_bit[ATT_MAX_COMMITTEES + 1], s_start[ATT_MAX_COMMITTEES], s_meta[2];
    __shared__ uint32_t s_warp[ATT_WRITE_THREADS / 32];
    __shared__ uint32_t s_sort[ATT_SORT_MAX];
    const uint32_t i = blockIdx.x, st = p.status[i];
    if (st != ATT_OK && st != ATT_UNKNOWN_VALIDATOR) return;
    const uint32_t koff = wr.key_off[i];
    const bool to_out = wr.out != nullptr, sort_here = to_out && !p.electra;
    if (koff == UINT32_MAX && !to_out) return;
    const uint32_t fixed = p.electra ? ATT_FIXED_ELECTRA : ATT_FIXED;
    const uint8_t* r = nullptr;
    uint32_t nb = 0, n_bits = 0;
    att_frame(p, i, r, nb, n_bits);   // framed and resolved by k_attestation_index_count already
    if (threadIdx.x == 0) {
        uint32_t ci = 0, n_seg = 0;
        att_committees(p, r, n_bits, ci, s_bit, s_start, n_seg);
        s_meta[0] = ci;
        s_meta[1] = n_seg;
    }
    __syncthreads();
    const uint64_t* sh = p.cache[s_meta[0]].shuffling;
    const uint32_t n_seg = s_meta[1], lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t o0 = to_out ? wr.out_off[i] : 0;
    uint32_t base = 0;
    for (uint32_t b0 = 0; b0 < n_bits; b0 += ATT_WRITE_THREADS) {
        const uint32_t q = b0 + threadIdx.x;
        const bool set = q < n_bits && ((r[fixed + q / 8] >> (q % 8)) & 1);
        const uint32_t v = set ? (uint32_t)sh[att_position(s_bit, s_start, n_seg, q)] : 0;
        const uint32_t ballot = __ballot_sync(0xffffffffu, set);
        if (lane == 0) s_warp[wid] = __popc(ballot);
        __syncthreads();
        uint32_t before = 0, total = 0;
#pragma unroll
        for (int k = 0; k < ATT_WRITE_THREADS / 32; k++) {
            const uint32_t c = s_warp[k];
            before += k < (int)wid ? c : 0;
            total += c;
        }
        const uint32_t pos = base + before + __popc(ballot & ((1u << lane) - 1));
        if (set) {
            if (koff != UINT32_MAX) wr.keys[koff + pos] = v;
            if (sort_here) s_sort[pos] = v;
            else if (to_out) wr.out[o0 + pos] = v;
        }
        base += total;
        __syncthreads();
    }
    if (!sort_here) return;
    // sort_unstable: a bitonic sort over the next power of two, padded with the largest key
    uint32_t m = 1;
    while (m < base) m <<= 1;
    for (uint32_t k = base + threadIdx.x; k < m; k += ATT_WRITE_THREADS) s_sort[k] = UINT32_MAX;
    __syncthreads();
    for (uint32_t size = 2; size <= m; size <<= 1)
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < m / 2; t += ATT_WRITE_THREADS) {
                const uint32_t lo = 2 * stride * (t / stride) + (t % stride), hi = lo + stride;
                const uint32_t a = s_sort[lo], b = s_sort[hi];
                if ((a > b) == ((lo & size) == 0)) { s_sort[lo] = b; s_sort[hi] = a; }
            }
            __syncthreads();
        }
    for (uint32_t k = threadIdx.x; k < base; k += ATT_WRITE_THREADS) wr.out[o0 + k] = s_sort[k];
}

}  // namespace lhb200
