// merkle.cuh — SSZ merkleization kernels (sm_90a).  See DESIGN.md §"Tree-hash path".
//
// Kernel inventory (SURVEY.md §2d K1-K3):
//   k_hash_pairs ........ n independent hash32_concat (ethereum_hashing::hash32_concat batch)
//   k_validator_roots ... 121-byte SSZ Validator -> 32-byte root (8 hashes / validator, validator.rs:25-35)
//   k_record_roots ...... small fixed records: 48-B pubkey (bls/src/macros.rs:18-25), 72-B Eth1Data, 192-B DepositRequest
//   k_merkle_reduce ..... multi-segment tile reduce: every CTA folds up to 2^11 chunks of one segment
//                         (up to 11 tree levels) and writes one node; virtual zero padding via ZERO_HASHES
//   k_hash_program ...... small DAG interpreter (zero ladders, mix_in_length, small containers, top tree)
#pragma once
#include "sha256.cuh"

namespace lhb200 {

constexpr int MAX_ZERO_DEPTH = 64;
// ZERO_HASHES[d] in word form (merkle_proof/src/lib.rs:166).  Filled by k_init_zero_hashes at init.
__device__ uint32_t g_zero_words[MAX_ZERO_DEPTH + 1][8];

__global__ void k_init_zero_hashes() {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t cur[8];
#pragma unroll
    for (int i = 0; i < 8; i++) cur[i] = 0;
    for (int d = 0; d <= MAX_ZERO_DEPTH; d++) {
        for (int i = 0; i < 8; i++) g_zero_words[d][i] = cur[i];
        hash_pair(cur, cur, cur);
    }
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_hash_pairs(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                    uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t l[8], r[8], o[8];
    load_chunk(in + 64 * i, l);
    load_chunk(in + 64 * i + 32, r);
    hash_pair_inl(l, r, o);
    store_chunk(out + 32 * i, o);
}

// ---------------------------------------------------------------------------------------------
// Validator roots.  One CTA stages 256 validators (30 976 contiguous bytes, 16-B aligned because the
// staged list base is 256-B aligned and 256*121 is a multiple of 16) into shared memory with coalesced
// uint4 loads, then each thread builds its validator's 8 leaves and folds them (8 hashes).
constexpr int VAL_SSZ = 121;
constexpr int VAL_PER_CTA = 256;

__device__ __forceinline__ uint32_t be_word(const uint8_t* p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}
// little-endian u64 field -> first two SHA words of its (zero padded) chunk
__device__ __forceinline__ void le64_words(const uint8_t* p, uint32_t& w0, uint32_t& w1) {
    w0 = be_word(p);
    w1 = be_word(p + 4);
}

// hash_tree_root of one 121-byte Validator record (validator.rs:25-35): 8 leaves, 8 hashes.  `v`: shared or global.
__device__ __forceinline__ void validator_root_words(const uint8_t* v, uint32_t h01[8]) {
    uint32_t a[8], b[8], h23[8];
    // leaf0 = H(pubkey[0:32] || pubkey[32:48] || 0^16)
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = be_word(v + 4 * i);
#pragma unroll
    for (int i = 0; i < 4; i++) b[i] = be_word(v + 32 + 4 * i);
    b[4] = b[5] = b[6] = b[7] = 0;
    hash_pair(a, b, a);
    // leaf1 = withdrawal_credentials
#pragma unroll
    for (int i = 0; i < 8; i++) b[i] = be_word(v + 48 + 4 * i);
    hash_pair(a, b, h01);
    // leaf2 = effective_balance, leaf3 = slashed
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = b[i] = 0;
    le64_words(v + 80, a[0], a[1]);
    b[0] = (uint32_t)v[88] << 24;
    hash_pair(a, b, h23);
    hash_pair(h01, h23, h01);  // h0123
    // leaf4..7 = activation_eligibility, activation, exit, withdrawable epochs
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = b[i] = 0;
    le64_words(v + 89, a[0], a[1]);
    le64_words(v + 97, b[0], b[1]);
    hash_pair(a, b, h23);  // h45
    a[0] = a[1] = b[0] = b[1] = 0;
    le64_words(v + 105, a[0], a[1]);
    le64_words(v + 113, b[0], b[1]);
    hash_pair(a, b, a);      // h67
    hash_pair(h23, a, h23);  // h4567
    hash_pair(h01, h23, h01);
}

__global__ void __launch_bounds__(VAL_PER_CTA) k_validator_roots(const uint8_t* __restrict__ ssz, uint64_t n,
                                                                 uint8_t* __restrict__ out) {
    __shared__ __align__(16) uint8_t sm[VAL_PER_CTA * VAL_SSZ];
    const uint64_t first = (uint64_t)blockIdx.x * VAL_PER_CTA;
    const uint64_t cnt = min((uint64_t)VAL_PER_CTA, n - first);
    const uint32_t nbytes = (uint32_t)cnt * VAL_SSZ;
    const uint8_t* src = ssz + first * VAL_SSZ;
    {
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        uint4* d4 = reinterpret_cast<uint4*>(sm);
        const uint32_t nvec = nbytes / 16;
        for (uint32_t i = threadIdx.x; i < nvec; i += VAL_PER_CTA) d4[i] = __ldg(s4 + i);
        for (uint32_t i = nvec * 16 + threadIdx.x; i < nbytes; i += VAL_PER_CTA) sm[i] = src[i];
    }
    __syncthreads();
    if (threadIdx.x >= cnt) return;
    const uint8_t* v = sm + threadIdx.x * VAL_SSZ;

    uint32_t h01[8];
    validator_root_words(v, h01);
    store_chunk(out + 32 * (first + threadIdx.x), h01);
}

// ---------------------------------------------------------------------------------------------
// Small fixed-size records -> roots.  kind 0: 48-byte pubkey.  kind 1: 72-byte Eth1Data {H256,u64,H256}.
// kind 2: 16-byte {u64, u64} (PendingBalanceDeposit, PendingConsolidation).  kind 3: 24-byte {u64, u64, u64}
// (PendingPartialWithdrawal): the Electra state lists, beacon_state.rs:515-525.  kind 4: 192-byte DepositRequest
// {pubkey, withdrawal_credentials, amount, signature, index} (deposit_request.rs:23-29), 10 hashes.  kind 5: 64-byte
// HistoricalSummary {H256, H256} (historical_summary.rs).  Loads are bytewise, so records may sit at any byte offset
// (the block path reads them straight from the staged SSZ blob).
constexpr int REC_PUBKEY = 0, REC_ETH1_DATA = 1, REC_U64_PAIR = 2, REC_U64_TRIPLE = 3, REC_DEPOSIT_REQUEST = 4,
              REC_HISTORICAL_SUMMARY = 5;
__host__ __device__ constexpr uint32_t record_bytes(int kind) {
    return kind == REC_PUBKEY ? 48 : kind == REC_ETH1_DATA ? 72 : kind == REC_U64_PAIR ? 16
         : kind == REC_U64_TRIPLE ? 24 : kind == REC_DEPOSIT_REQUEST ? 192 : 64;
}

// hash_tree_root of the record of `kind` at p.  Shared by k_record_roots (cold) and k_tree_update_level (warm).
__device__ __forceinline__ void record_root_words(const uint8_t* p, int kind, uint32_t a[8]) {
    uint32_t b[8];
    if (kind == REC_DEPOSIT_REQUEST) {
        uint32_t c[8];
        for (int k = 0; k < 8; k++) a[k] = be_word(p + 4 * k);
        for (int k = 0; k < 4; k++) b[k] = be_word(p + 32 + 4 * k);
        b[4] = b[5] = b[6] = b[7] = 0;
        hash_pair(a, b, a);                       // pubkey
        for (int k = 0; k < 8; k++) b[k] = be_word(p + 48 + 4 * k);
        hash_pair(a, b, a);                       // H(pubkey, withdrawal_credentials)
        for (int k = 0; k < 8; k++) b[k] = be_word(p + 88 + 4 * k);
        for (int k = 0; k < 8; k++) c[k] = be_word(p + 120 + 4 * k);
        hash_pair(b, c, b);                       // signature chunks 0, 1
        for (int k = 0; k < 8; k++) c[k] = be_word(p + 152 + 4 * k);
        hash_pair(c, g_zero_words[0], c);         // signature chunk 2, zero chunk
        hash_pair(b, c, b);                       // signature root
        for (int k = 0; k < 8; k++) c[k] = 0;
        le64_words(p + 80, c[0], c[1]);
        hash_pair(c, b, c);                       // H(amount, signature)
        hash_pair(a, c, a);                       // fields 0..3
        for (int k = 0; k < 8; k++) c[k] = 0;
        le64_words(p + 184, c[0], c[1]);
        hash_pair(c, g_zero_words[0], c);         // H(index, zero chunk)
        hash_pair(c, g_zero_words[1], c);         // fields 4..7
        hash_pair(a, c, a);
    } else if (kind == REC_PUBKEY) {
        for (int k = 0; k < 8; k++) a[k] = be_word(p + 4 * k);
        for (int k = 0; k < 4; k++) b[k] = be_word(p + 32 + 4 * k);
        b[4] = b[5] = b[6] = b[7] = 0;
        hash_pair(a, b, a);
    } else if (kind == REC_U64_PAIR || kind == REC_U64_TRIPLE) {
        for (int k = 0; k < 8; k++) a[k] = b[k] = 0;
        le64_words(p, a[0], a[1]);
        le64_words(p + 8, b[0], b[1]);
        hash_pair(a, b, a);                       // H(field 0, field 1)
        if (kind == REC_U64_TRIPLE) {
            uint32_t c[8];
            for (int k = 0; k < 8; k++) c[k] = b[k] = 0;
            le64_words(p + 16, c[0], c[1]);
            hash_pair(c, b, c);                   // H(field 2, zero chunk)
            hash_pair(a, c, a);
        }
    } else if (kind == REC_HISTORICAL_SUMMARY) {
        for (int k = 0; k < 8; k++) a[k] = be_word(p + 4 * k);
        for (int k = 0; k < 8; k++) b[k] = be_word(p + 32 + 4 * k);
        hash_pair(a, b, a);
    } else {
        uint32_t c[8];
        for (int k = 0; k < 8; k++) a[k] = be_word(p + 4 * k);
        for (int k = 0; k < 8; k++) b[k] = 0;
        le64_words(p + 32, b[0], b[1]);
        hash_pair(a, b, a);  // H(deposit_root, deposit_count)
        for (int k = 0; k < 8; k++) c[k] = be_word(p + 40 + 4 * k);
        for (int k = 0; k < 8; k++) b[k] = 0;
        hash_pair(c, b, c);  // H(block_hash, zero chunk)
        hash_pair(a, c, a);
    }
}

__global__ void __launch_bounds__(128) k_record_roots(const uint8_t* __restrict__ in, uint64_t n, int kind,
                                                      uint8_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t a[8];
    record_root_words(in + (uint64_t)record_bytes(kind) * i, kind, a);
    store_chunk(out + 32 * i, a);
}

// ---------------------------------------------------------------------------------------------
// Phase0 PendingAttestation (pending_attestation.rs:25-32): {aggregation_bits: Bitlist[2048] behind the offset at 0,
// data: AttestationData (128 B at 4), inclusion_delay: u64 at 132, proposer_index: u64 at 140}, then the bitlist bytes.
// A phase0 BeaconState holds two List[PendingAttestation, 4096] (fields 15 and 16).  k_pending_attestation_roots runs
// one thread per slot of a 4096-slot root array per list, reading the records straight from the staged list bytes
// through their offset table: slot i < n gets record i's root (19 hashes: 8 for the bitlist with its length, 8 for the
// AttestationData, 3 for the record), slots n.. get zero chunks, so that the full 4096-leaf tree over the array is the
// list's data root at every length.  The host has checked offsets, record sizes, delimiters and bit counts, and no patch
// reaches a staged list; even so a record whose offsets do not frame 149 to 405 bytes inside the list gets a zero chunk,
// so that no byte of a list can steer a read outside it.
constexpr uint32_t PENDING_FIXED = 148, MAX_PENDING = 4096, PENDING_HASHES = 19;
struct PendingSeg {
    const uint8_t* in;   // the list's SSZ bytes: offset table, then the records
    uint8_t* out;        // MAX_PENDING root chunks
    uint64_t bytes;
    uint32_t n;          // records
};
constexpr int MAX_PENDING_SEGS = 2;
struct PendingTable {
    int n;
    PendingSeg s[MAX_PENDING_SEGS];
};

__device__ __forceinline__ uint32_t le_u32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
// Chunk c of a bitlist's bits without its delimiter: the nb bytes at b, zero past them, the last byte's highest set
// bit cleared.
__device__ __forceinline__ void bitlist_chunk(const uint8_t* b, uint32_t nb, uint32_t c, uint32_t w[8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        uint32_t x = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t j = 32 * c + 4 * k + q;
            uint32_t v = j < nb ? b[j] : 0;
            if (j + 1 == nb && v) v &= ~(0x80000000u >> __clz(v));
            x = (x << 8) | v;
        }
        w[k] = x;
    }
}
// 8-byte little-endian field -> its chunk
__device__ __forceinline__ void u64_chunk(const uint8_t* p, uint32_t w[8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = 0;
    le64_words(p, w[0], w[1]);
}
__device__ __forceinline__ void h256_chunk(const uint8_t* p, uint32_t w[8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = be_word(p + 4 * k);
}
// hash_tree_root of the PendingAttestation of `len` bytes at r
__device__ __forceinline__ void pending_attestation_root_words(const uint8_t* r, uint32_t len, uint32_t h[8]) {
    uint32_t a[8], b[8], t[8];
    // aggregation_bits: 8 chunks (2048 bits), then the bit count mixed in
    const uint8_t* bits = r + PENDING_FIXED;
    const uint32_t nb = len - PENDING_FIXED;
    bitlist_chunk(bits, nb, 0, a); bitlist_chunk(bits, nb, 1, b); hash_pair(a, b, h);
    bitlist_chunk(bits, nb, 2, a); bitlist_chunk(bits, nb, 3, b); hash_pair(a, b, a); hash_pair(h, a, h);
    bitlist_chunk(bits, nb, 4, a); bitlist_chunk(bits, nb, 5, b); hash_pair(a, b, t);
    bitlist_chunk(bits, nb, 6, a); bitlist_chunk(bits, nb, 7, b); hash_pair(a, b, a); hash_pair(t, a, t);
    hash_pair(h, t, h);
    const uint32_t last = bits[nb - 1];
    const uint32_t n_bits = 8 * (nb - 1) + 31 - __clz(last);
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = 0;
    a[0] = bswap32(n_bits);
    hash_pair(h, a, h);
    // AttestationData {slot, index, beacon_block_root, source, target}: 8 leaves
    const uint8_t* d = r + 4;
    u64_chunk(d, a); u64_chunk(d + 8, b); hash_pair(a, b, t);                        // H(slot, index)
    u64_chunk(d + 48, a); h256_chunk(d + 56, b); hash_pair(a, b, b);                 // source
    h256_chunk(d + 16, a); hash_pair(a, b, a);                                       // H(beacon_block_root, source)
    hash_pair(t, a, t);
    u64_chunk(d + 88, a); h256_chunk(d + 96, b); hash_pair(a, b, a);                 // target
    hash_pair(a, g_zero_words[0], a);
    hash_pair(a, g_zero_words[1], a);
    hash_pair(t, a, t);
    // the record: {aggregation_bits, data, inclusion_delay, proposer_index}
    hash_pair(h, t, h);
    u64_chunk(r + 132, a); u64_chunk(r + 140, b); hash_pair(a, b, a);
    hash_pair(h, a, h);
}

__global__ void __launch_bounds__(128) k_pending_attestation_roots(const __grid_constant__ PendingTable tab) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = g / MAX_PENDING, i = g % MAX_PENDING;
    if ((int)s >= tab.n) return;
    const PendingSeg& seg = tab.s[s];
    uint32_t h[8];
    const uint64_t o0 = i < seg.n ? le_u32(seg.in + 4 * i) : 0;
    const uint64_t o1 = i + 1 < seg.n ? le_u32(seg.in + 4 * i + 4) : seg.bytes;
    if (i < seg.n && o0 >= 4ull * seg.n && o1 <= seg.bytes && o1 >= o0 + PENDING_FIXED + 1 &&
        o1 - o0 <= PENDING_FIXED + 257) {
        pending_attestation_root_words(seg.in + o0, (uint32_t)(o1 - o0), h);
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) h[k] = 0;
    }
    store_chunk(seg.out + 32ull * i, h);
}

// ---------------------------------------------------------------------------------------------
// Multi-segment tile reduce.
struct MerkleSeg {
    const uint8_t* in;   // n_in chunks (32 B each, 16-B aligned); roots of height-`level_in` subtrees
    uint8_t* out;        // ceil(n_in / 2^tile_log) chunks
    uint64_t n_in;
    uint32_t level_in;   // height of the input nodes above the segment's leaves (selects ZERO_HASHES row)
    uint32_t tile_log;   // levels folded by one CTA, 1..11
    uint32_t cta_begin;  // first CTA index serving this segment
    uint32_t n_tiles;
};
constexpr int MAX_SEGS = 24;
struct MerkleSegTable {
    int n;
    MerkleSeg s[MAX_SEGS];
};
constexpr int REDUCE_THREADS = 256;
constexpr int MAX_TILE_LOG = 11;  // 256 threads x 8 chunks

// fold (l, r) where the right node may be virtual padding
__device__ __forceinline__ void fold(uint32_t l[8], const uint32_t r[8], bool r_valid, uint32_t zlevel) {
    uint32_t rr[8];
#pragma unroll
    for (int i = 0; i < 8; i++) rr[i] = r_valid ? r[i] : g_zero_words[zlevel][i];
    hash_pair(l, rr, l);
}

__global__ void __launch_bounds__(REDUCE_THREADS) k_merkle_reduce(const __grid_constant__ MerkleSegTable tab) {
    __shared__ uint32_t sm[2][REDUCE_THREADS][8];
    int si = 0;
#pragma unroll 1
    for (int k = 1; k < tab.n; k++)
        if (blockIdx.x >= tab.s[k].cta_begin) si = k;
    const MerkleSeg& sg = tab.s[si];
    const uint32_t tile = blockIdx.x - sg.cta_begin;
    const uint32_t tl = sg.tile_log;
    const uint32_t t = tl < 3 ? tl : 3;  // levels folded privately by each thread
    const uint32_t nthr_a = 1u << (tl - t);
    const uint64_t n_in = sg.n_in;
    const uint32_t tid = threadIdx.x;

    // ---- phase A: each active thread folds 2^t consecutive chunks straight from global memory
    if (tid < nthr_a) {
        const uint64_t base = ((uint64_t)tile << tl) + ((uint64_t)tid << t);
        const uint32_t cnt = base >= n_in ? 0u : (uint32_t)min((uint64_t)(1u << t), n_in - base);
        if (cnt > 0) {
            uint32_t nd[4][8];
            uint32_t c = cnt;
            if (t == 0) {
                load_chunk(sg.in + 32 * base, nd[0]);
            } else {
#pragma unroll
                for (int p = 0; p < 4; p++) {
                    if (p < (1 << (t - 1)) && 2u * p < c) {
                        uint32_t r[8];
                        load_chunk(sg.in + 32 * (base + 2 * p), nd[p]);
                        const bool rv = 2u * p + 1 < c;
                        if (rv) load_chunk(sg.in + 32 * (base + 2 * p + 1), r);
                        fold(nd[p], r, rv, sg.level_in);
                    }
                }
                c = (c + 1) >> 1;
                if (t >= 2) {
#pragma unroll
                    for (int p = 0; p < 2; p++)
                        if (p < (1 << (t - 2)) && 2u * p < c) {
                            if (p) {
#pragma unroll
                                for (int i = 0; i < 8; i++) nd[1][i] = nd[2][i];
                            }
                            fold(nd[p], nd[2 * p + 1], 2u * p + 1 < c, sg.level_in + 1);
                        }
                    c = (c + 1) >> 1;
                }
                if (t >= 3) fold(nd[0], nd[1], 1 < c, sg.level_in + 2);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) sm[0][tid][i] = nd[0][i];
        }
    }
    // ---- phase B: remaining tl - t levels through shared memory, compacting active threads each level
    int cur = 0;
    uint32_t width = nthr_a;                   // nodes of this tile at the current level
    uint32_t lvl = t;                          // level (relative to segment input) of the nodes in sm[cur]
    while (width > 1) {
        __syncthreads();
        const uint32_t half = width >> 1;
        // number of valid nodes at `lvl` over the whole segment
        const uint64_t valid_total = (n_in + ((1ull << lvl) - 1)) >> lvl;
        if (tid < half) {
            const uint64_t gl = (uint64_t)tile * width + 2 * tid;  // global index of the left child
            if (gl < valid_total) {
                uint32_t l[8], r[8];
#pragma unroll
                for (int i = 0; i < 8; i++) { l[i] = sm[cur][2 * tid][i]; r[i] = sm[cur][2 * tid + 1][i]; }
                fold(l, r, gl + 1 < valid_total, sg.level_in + lvl);
#pragma unroll
                for (int i = 0; i < 8; i++) sm[cur ^ 1][tid][i] = l[i];
            }
        }
        cur ^= 1;
        width = half;
        lvl++;
    }
    __syncthreads();
    if (tid == 0) {
        const uint64_t valid_total = (n_in + ((1ull << tl) - 1)) >> tl;
        if (tile < valid_total) {
            uint32_t o[8];
#pragma unroll
            for (int i = 0; i < 8; i++) o[i] = sm[cur][0][i];
            store_chunk(sg.out + 32ull * tile, o);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Hash program: a DAG of hash32_concat ops over 32-byte nodes anywhere in device memory, executed wave by
// wave by one CTA.  Operand with bit 63 clear: device address of a 16-B aligned 32-byte node.
// Operand with bit 63 set: ZERO_HASHES[operand & 0xff].
struct HashOp {
    uint64_t dst, a, b;
};
constexpr uint64_t OP_ZERO_FLAG = 1ull << 63;
constexpr int PROG_THREADS = 128;

__device__ __forceinline__ void load_operand(uint64_t op, uint32_t w[8]) {
    if (op & OP_ZERO_FLAG) {
        const uint32_t d = (uint32_t)(op & 0xff);
        for (int i = 0; i < 8; i++) w[i] = g_zero_words[d][i];
    } else {
        // plain (coherent) loads: nodes may have been written earlier in this same launch
        const uint4* p = reinterpret_cast<const uint4*>(op);
        uint4 x = p[0], y = p[1];
        w[0] = bswap32(x.x); w[1] = bswap32(x.y); w[2] = bswap32(x.z); w[3] = bswap32(x.w);
        w[4] = bswap32(y.x); w[5] = bswap32(y.y); w[6] = bswap32(y.z); w[7] = bswap32(y.w);
    }
}

__global__ void __launch_bounds__(PROG_THREADS) k_hash_program(const HashOp* __restrict__ ops,
                                                               const int32_t* __restrict__ wave_begin,
                                                               int n_waves) {
    for (int w = 0; w < n_waves; w++) {
        const int lo = wave_begin[w], hi = wave_begin[w + 1];
        for (int k = lo + threadIdx.x; k < hi; k += PROG_THREADS) {
            const HashOp op = ops[k];
            uint32_t l[8], r[8];
            load_operand(op.a, l);
            load_operand(op.b, r);
            hash_pair(l, r, l);
            store_chunk(reinterpret_cast<uint8_t*>(op.dst), l);
        }
        __syncthreads();
    }
}

// One wave of a hash program spread over the whole grid (used when a wave is too wide for one CTA: block batches).
__global__ void __launch_bounds__(PROG_THREADS) k_hash_ops(const HashOp* __restrict__ ops, int n) {
    const int k = blockIdx.x * PROG_THREADS + threadIdx.x;
    if (k >= n) return;
    const HashOp op = ops[k];
    uint32_t l[8], r[8];
    load_operand(op.a, l);
    load_operand(op.b, r);
    hash_pair(l, r, l);
    store_chunk(reinterpret_cast<uint8_t*>(op.dst), l);
}

// ---------------------------------------------------------------------------------------------
// Device-resident Merkle trees for the warm path (SURVEY.md §8f-3; the reference's steady state is the tree-hash
// cache: BeaconState::update_tree_hash_cache re-hashes only dirty paths, beacon_state.rs:2031-2038,2459-2481).
// Every big list of a resident state keeps ALL its levels; after lhb200_state_patch marks leaves dirty, one CTA per
// tree re-hashes just the paths above them, level by level.
struct TreeDev {
    const uint8_t* src;     // kind 0: the 121-byte validator records, kind >= 2: the records (leaf roots are recomputed)
    uint8_t* lvl[41];       // lvl[0] = leaf chunks, lvl[top] = one node
    uint64_t n_leaves;      // current leaf count (a resizable list follows its length)
    uint32_t top;           // ceil_log2(n_leaves)
    uint32_t kind;          // 0: validators, 1: chunks are the data, 2 + k: records of k_record_roots kind k
    uint8_t* top_dst;       // where the plan's tail program reads this list's data root (null: resizable list)
    const uint32_t* dirty;  // sorted, unique leaf indices
    uint32_t n_dirty;
    uint32_t limit_depth;   // resizable list: chunk-tree depth of its limit
    uint64_t length;        // resizable list: item count mixed into its root
    uint8_t* field_dst;     // resizable list: where k_list_finish writes the field root
};
constexpr uint32_t TREE_VALIDATORS = 0, TREE_CHUNKS = 1, TREE_RECORDS = 2;

// out[i] = H(in[2i], in[2i+1] or ZERO[zlevel]) for i < ceil(n_in / 2)   (full build of one level)
__global__ void __launch_bounds__(256) k_tree_level(const uint8_t* __restrict__ in, uint64_t n_in,
                                                    uint8_t* __restrict__ out, uint32_t zlevel) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (2 * i >= n_in) return;
    uint32_t l[8], r[8];
    load_chunk(in + 64 * i, l);
    const bool rv = 2 * i + 1 < n_in;
    if (rv) load_chunk(in + 64 * i + 32, r);
    fold(l, r, rv, zlevel);
    store_chunk(out + 32 * i, l);
}

// One level of the dirty-path update for ALL trees of a state: blockIdx.y = tree, one thread per dirty leaf.
// level < 0: recompute the leaf roots of dirty validators / records.  Otherwise the first dirty leaf under each parent
// at `level + 1` hashes that parent from its two children at `level`; a child past the current length is the zero
// node of its height, so after a truncation the path of the new last leaf rebuilds the right edge.
__global__ void __launch_bounds__(256) k_tree_update_level(const TreeDev* __restrict__ trees, int level) {
    const TreeDev& t = trees[blockIdx.y];
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= t.n_dirty) return;
    if (level < 0) {
        if (t.kind == TREE_CHUNKS) return;
        const uint32_t i = t.dirty[j];
        uint32_t w[8];
        if (t.kind == TREE_VALIDATORS) validator_root_words(t.src + (uint64_t)VAL_SSZ * i, w);
        else record_root_words(t.src + (uint64_t)record_bytes(t.kind - TREE_RECORDS) * i, t.kind - TREE_RECORDS, w);
        store_chunk(t.lvl[0] + 32ull * i, w);
        return;
    }
    const uint32_t l = (uint32_t)level;
    if (l >= t.top) return;
    const uint32_t p = t.dirty[j] >> (l + 1);
    if (j != 0 && (t.dirty[j - 1] >> (l + 1)) == p) return;
    const uint64_t n_l = (t.n_leaves + ((1ull << l) - 1)) >> l;   // nodes at this level
    uint32_t a[8], b[8];
    load_operand(reinterpret_cast<uint64_t>(t.lvl[l] + 64ull * p), a);
    const bool rv = 2ull * p + 1 < n_l;
    if (rv) load_operand(reinterpret_cast<uint64_t>(t.lvl[l] + 64ull * p + 32), b);
    fold(a, b, rv, l);
    store_chunk(t.lvl[l + 1] + 32ull * p, a);
    if (l + 1 == t.top && t.top_dst) store_chunk(t.top_dst, a);
}

// Finishing step of resizable lists: one thread per list.  Field root = mix_in_length(data root laddered from the
// current top to the limit depth with ZERO_HASHES, length); an empty list is ZERO_HASHES[limit depth] mixed with 0.
constexpr int MAX_FINISH = 16;
struct FinishTable {
    uint32_t n;
    uint32_t tree[MAX_FINISH];   // indices into the TreeDev array
};
__global__ void __launch_bounds__(32) k_list_finish(const TreeDev* __restrict__ trees,
                                                    const __grid_constant__ FinishTable tab) {
    if (threadIdx.x >= tab.n) return;
    const TreeDev& t = trees[tab.tree[threadIdx.x]];
    uint32_t r[8];
    if (t.n_leaves == 0) {
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = g_zero_words[t.limit_depth][i];
    } else {
        load_operand(reinterpret_cast<uint64_t>(t.lvl[t.top]), r);
        for (uint32_t l = t.top; l < t.limit_depth; l++) hash_pair(r, g_zero_words[l], r);
    }
    uint32_t len[8] = {bswap32((uint32_t)t.length), bswap32((uint32_t)(t.length >> 32)), 0, 0, 0, 0, 0, 0};
    hash_pair(r, len, r);
    store_chunk(t.field_dst, r);
}

// Scatter a batch of same-length byte patches from one staged blob into resident buffers: one warp per patch.
struct ScatterOp {
    uint8_t* dst;
    uint32_t len;
    uint32_t blob_off;
};
__global__ void __launch_bounds__(256) k_scatter_bytes(const ScatterOp* __restrict__ ops, uint32_t n,
                                                       const uint8_t* __restrict__ blob) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    const ScatterOp op = ops[w];
    for (uint32_t i = lane; i < op.len; i += 32) op.dst[i] = blob[op.blob_off + i];
}

// Device-to-device copy of many ranges in one launch (lhb200_state_clone).  Every range is a whole number of 16-byte
// words at 16-byte aligned addresses; word[k] = 16-byte words of ranges [0, k), word[n] = the total.  Grid-stride over
// the total: each thread finds the range of its first word by binary search over `word` and walks forward from there,
// since its later words only lie in the same or later ranges.
struct CopyRange {
    uint8_t* dst;
    const uint8_t* src;
    uint64_t bytes;   // multiple of 16
};
__global__ void __launch_bounds__(256) k_copy_ranges(const CopyRange* __restrict__ ranges,
                                                     const uint64_t* __restrict__ word, uint32_t n) {
    const uint64_t total = word[n], stride = (uint64_t)gridDim.x * blockDim.x;
    uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= total) return;
    uint32_t lo = 0, hi = n;   // word[lo] <= w < word[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (word[mid] <= w) lo = mid; else hi = mid;
    }
    for (; w < total; w += stride) {
        while (word[lo + 1] <= w) lo++;
        const uint64_t o = (w - word[lo]) * 16;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(ranges[lo].src + o));
        *reinterpret_cast<uint4*>(ranges[lo].dst + o) = v;
    }
}

// Merkle branches by generalized index (lhb200_state_proofs, lhb200_beacon_block_body_proofs).  The host resolves each
// proof down to the tree it enters (or to its end) and lists the siblings above that point once per distinct path
// prefix, as ProofSrc entries.  One thread per output sibling: it finds its proof by binary search over the prefix
// sums of the branch depths (first[k] = siblings of proofs [0, k)), reads the sibling and stores it with uint4 writes, so
// consecutive threads write consecutive 32-byte entries of one branch.  A sibling that is a plain device address is
// copied with uint4 loads: like every hash-program operand (load_operand) it must be 16-byte aligned, and so must a new
// kind of operand source (level arrays, node pool, literals, leaf and item outputs all are).
struct ProofTree {            // levels of one tree: lvl[l] holds ceil(n_leaves / 2^l) nodes, the rest are zero nodes
    const uint8_t* lvl[41];
    uint64_t n_leaves;
};
struct ProofSrc {             // operand `op` (a device address or OP_ZERO_FLAG | level), hashed with ZERO_HASHES[l] for
    uint64_t op;              // l in [from, to): the left spine node of a list above its current top
    uint32_t from, to;
};
struct ProofDesc {
    uint64_t node;            // index of the proven node at level `level` of tree `tree`
    uint32_t tree, level;
    uint32_t n_tree;          // siblings 0 .. n_tree-1 (bottom-up) lie in the tree, the rest are srcs[src ..]
    uint32_t src;
};
__global__ void __launch_bounds__(256) k_proof_branches(const ProofDesc* __restrict__ proofs,
                                                        const uint64_t* __restrict__ first, uint32_t n,
                                                        const ProofTree* __restrict__ trees,
                                                        const ProofSrc* __restrict__ srcs, uint8_t* __restrict__ out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= first[n]) return;
    uint32_t lo = 0, hi = n;   // first[lo] <= t < first[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (first[mid] <= t) lo = mid; else hi = mid;
    }
    const ProofDesc p = proofs[lo];
    const uint32_t j = (uint32_t)(t - first[lo]);
    uint64_t op;
    uint32_t from = 0, to = 0;
    if (j < p.n_tree) {
        const ProofTree& tr = trees[p.tree];
        const uint32_t l = p.level + j;
        const uint64_t idx = (p.node >> j) ^ 1, cnt = (tr.n_leaves + ((1ull << l) - 1)) >> l;
        op = idx < cnt ? reinterpret_cast<uint64_t>(tr.lvl[l] + 32 * idx) : (OP_ZERO_FLAG | l);
    } else {
        const ProofSrc s = srcs[p.src + (j - p.n_tree)];
        op = s.op; from = s.from; to = s.to;
    }
    uint4* dst = reinterpret_cast<uint4*>(out + 32 * t);
    if (!(op & OP_ZERO_FLAG) && from == to) {
        const uint4* s = reinterpret_cast<const uint4*>(op);
        dst[0] = s[0];
        dst[1] = s[1];
        return;
    }
    uint32_t w[8];
    load_operand(op, w);
    for (uint32_t l = from; l < to; l++) hash_pair(w, g_zero_words[l], w);
    store_chunk(out + 32 * t, w);
}

// ---------------------------------------------------------------------------------------------
// Byte items: hash_tree_root of packed byte strings that sit at ARBITRARY byte offsets inside an SSZ blob
// (transactions, signatures, pubkeys, bitlists, index lists, proofs ... of a BeaconBlock):
//     root = merkleize(pack(bytes), limit = 2^depth) [ mixed in with `length` ]
// One CTA per item.  256-chunk tiles are folded through shared memory; tile roots are combined by a binary-counter
// stack (the streaming MerkleHasher shape, naive_aggregation_pool.rs:46-55) and the right-sparse ladder up to `depth`
// uses ZERO_HASHES, so a ByteList[2^30] costs its data hashes + <= 25 ladder hashes.
struct ByteItem {
    const uint8_t* src;   // first byte (any alignment); the buffer is readable 8 bytes past the end
    uint64_t nbytes;      // bytes that belong to the item (<= 32 << depth)
    uint8_t* out;         // 32-byte root (16-B aligned)
    uint64_t length;      // value mixed in when flags & 1
    uint32_t depth;       // limit = 2^depth chunks
    uint32_t flags;       // bit0: mix_in_length; bits 8..15: AND-mask applied to the item's last byte (bitlist delimiter)
};
constexpr int ITEM_THREADS = 128;
constexpr int ITEM_TILE_LOG = 8;

// chunk `c` of the item as 8 big-endian SHA words; bytes at or past nbytes read as zero
__device__ __forceinline__ void load_item_chunk(const ByteItem& it, uint64_t c, uint32_t w[8]) {
    const uint64_t off = 32 * c;
    const uintptr_t a = reinterpret_cast<uintptr_t>(it.src) + off;
    const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const uint32_t sh = 8 * (uint32_t)(a & 3);
    const uint64_t rem = it.nbytes - off;  // > 0 by construction
    const uint32_t mask = (it.flags >> 8) & 0xff;
    uint32_t lo = q[0];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint32_t v = 0;
        if (4u * i < rem) {
            const uint32_t hi = q[i + 1];
            v = __funnelshift_r(lo, hi, sh);  // little-endian bytes [4i, 4i+4)
            lo = hi;
            const uint64_t left = rem - 4u * i;  // valid bytes in this word (>= 1)
            if (left < 4) v &= (1u << (8 * (uint32_t)left)) - 1;
            if (left <= 4) v &= ~((uint32_t)(0xff ^ mask) << (8 * ((uint32_t)left - 1)));  // last byte of the item
        }
        w[i] = bswap32(v);
    }
}

__global__ void __launch_bounds__(ITEM_THREADS) k_byte_items(const ByteItem* __restrict__ items) {
    __shared__ uint32_t sm[2][ITEM_THREADS][8];
    __shared__ uint32_t pending[40][8];  // thread 0's counter stack, one slot per height
    const ByteItem it = items[blockIdx.x];
    const uint32_t tid = threadIdx.x;
    const uint64_t n = (it.nbytes + 31) / 32;
    const uint32_t depth = it.depth;
    const uint32_t th = depth < ITEM_TILE_LOG ? depth : ITEM_TILE_LOG;  // height of a tile root
    const uint64_t n_tiles = (n + (1ull << th) - 1) >> th;
    uint64_t have = 0;  // bit h set <=> pending[h] holds a complete left subtree (thread 0)
    for (uint64_t tile = 0; tile < n_tiles; tile++) {
        const uint64_t base = tile << th;
        const uint32_t m = (uint32_t)min((uint64_t)(1u << th), n - base);  // valid chunks in this tile (>= 1)
        uint32_t width;  // nodes in sm[cur]
        int cur = 0;
        uint32_t lvl;
        if (th == 0) {
            if (tid == 0) load_item_chunk(it, base, sm[0][0]);
            width = 1; lvl = 0;
        } else {
            if (2 * tid < m) {
                uint32_t l[8], r[8];
                load_item_chunk(it, base + 2 * tid, l);
                const bool rv = 2 * tid + 1 < m;
                if (rv) load_item_chunk(it, base + 2 * tid + 1, r);
                fold(l, r, rv, 0);
#pragma unroll
                for (int i = 0; i < 8; i++) sm[0][tid][i] = l[i];
            }
            width = 1u << (th - 1); lvl = 1;
        }
        while (width > 1) {
            __syncthreads();
            const uint32_t half = width >> 1;
            const uint32_t valid = (m + (1u << lvl) - 1) >> lvl;
            if (tid < half && 2 * tid < valid) {
                uint32_t l[8], r[8];
#pragma unroll
                for (int i = 0; i < 8; i++) { l[i] = sm[cur][2 * tid][i]; r[i] = sm[cur][2 * tid + 1][i]; }
                fold(l, r, 2 * tid + 1 < valid, lvl);
#pragma unroll
                for (int i = 0; i < 8; i++) sm[cur ^ 1][tid][i] = l[i];
            }
            cur ^= 1;
            width = half;
            lvl++;
        }
        __syncthreads();
        if (tid == 0) {  // push the tile root (height th) onto the counter stack
            uint32_t node[8];
#pragma unroll
            for (int i = 0; i < 8; i++) node[i] = sm[cur][0][i];
            uint32_t h = th;
            while ((have >> h) & 1) {
                uint32_t l[8];
#pragma unroll
                for (int i = 0; i < 8; i++) l[i] = pending[h][i];
                hash_pair(l, node, node);
                have &= ~(1ull << h);
                h++;
            }
#pragma unroll
            for (int i = 0; i < 8; i++) pending[h][i] = node[i];
            have |= 1ull << h;
        }
        __syncthreads();
    }
    if (tid == 0) {
        uint32_t cur[8];
        bool has = false;
        for (uint32_t h = th; h < depth; h++) {
            if ((have >> h) & 1) {
                uint32_t l[8];
#pragma unroll
                for (int i = 0; i < 8; i++) l[i] = pending[h][i];
                fold(l, cur, has, h);
#pragma unroll
                for (int i = 0; i < 8; i++) cur[i] = l[i];
                has = true;
            } else if (has) {
                fold(cur, cur, false, h);
            }
        }
        if ((have >> depth) & 1) {
#pragma unroll
            for (int i = 0; i < 8; i++) cur[i] = pending[depth][i];
        } else if (!has) {
#pragma unroll
            for (int i = 0; i < 8; i++) cur[i] = g_zero_words[depth][i];
        }
        if (it.flags & 1) {
            uint32_t len[8] = {bswap32((uint32_t)it.length), bswap32((uint32_t)(it.length >> 32)), 0, 0, 0, 0, 0, 0};
            hash_pair(cur, len, cur);
        }
        store_chunk(it.out, cur);
    }
}

// verify_merkle_proof batch (merkle_proof/src/lib.rs:357-389): one thread folds one branch bottom-up.
__global__ void __launch_bounds__(128) k_verify_branches(const uint8_t* __restrict__ leaves,
                                                         const uint8_t* __restrict__ branches, uint32_t depth,
                                                         const uint64_t* __restrict__ indices,
                                                         const uint8_t* __restrict__ roots, uint64_t n,
                                                         uint8_t* __restrict__ ok) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t cur[8], sib[8];
    load_chunk(leaves + 32 * i, cur);
    const uint64_t idx = indices[i];
    for (uint32_t d = 0; d < depth; d++) {
        load_chunk(branches + 32 * (i * depth + d), sib);
        if ((idx >> d) & 1) hash_pair(sib, cur, cur);
        else hash_pair(cur, sib, cur);
    }
    load_chunk(roots + 32 * i, sib);
    bool eq = true;
    for (int k = 0; k < 8; k++) eq &= (cur[k] == sib[k]);
    ok[i] = eq ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// swap-or-not shuffle (consensus/swap_or_not_shuffle/src/shuffle_list.rs:79-160; SURVEY.md §8f-4).
// The reference sweeps the list in place round by round, hashing as it goes.  On the device the 90 rounds are
// flattened: every hash the sweep can need depends only on (seed, round, position >> 8), so ONE launch computes all
// pivots and ONE all `rounds x ceil(n/256)` source blocks; then each output index walks its 90 rounds through that
// bit table independently (compute_shuffled_index with lookups instead of hashes) and gathers / scatters its element.
__device__ __forceinline__ void shuffle_seed_hash(const uint8_t* seed, uint32_t round, bool with_pos, uint32_t pos,
                                                  uint8_t out[32]) {
    uint8_t buf[37];
    for (int i = 0; i < 32; i++) buf[i] = seed[i];
    buf[32] = (uint8_t)round;
    buf[33] = (uint8_t)pos; buf[34] = (uint8_t)(pos >> 8); buf[35] = (uint8_t)(pos >> 16); buf[36] = (uint8_t)(pos >> 24);
    sha256_short(buf, with_pos ? 37 : 33, out);
}
// pivots[r] = le64(H(seed || r)[0:8]) % n ; sources[r][b] = H(seed || r || le32(b))
__global__ void __launch_bounds__(128) k_shuffle_hashes(const uint8_t* __restrict__ seed, uint32_t rounds, uint64_t n,
                                                        uint32_t n_blocks, uint64_t* __restrict__ pivots,
                                                        uint8_t* __restrict__ sources) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)rounds * n_blocks;
    uint8_t d[32];
    if (t < rounds) {
        shuffle_seed_hash(seed, (uint32_t)t, false, 0, d);
        uint64_t v = 0;
        for (int k = 7; k >= 0; k--) v = (v << 8) | d[k];
        pivots[t] = v % n;
    }
    if (t < total) {
        const uint32_t r = (uint32_t)(t / n_blocks), b = (uint32_t)(t % n_blocks);
        shuffle_seed_hash(seed, r, true, b, d);
        for (int i = 0; i < 32; i++) sources[32 * t + i] = d[i];
    }
}
__global__ void __launch_bounds__(256) k_shuffle_permute(const uint64_t* __restrict__ in, uint64_t* __restrict__ out,
                                                         uint64_t n, uint32_t rounds, uint32_t n_blocks,
                                                         const uint64_t* __restrict__ pivots,
                                                         const uint8_t* __restrict__ sources, int forwards) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t index = i;
    for (uint32_t r = 0; r < rounds; r++) {
        const uint64_t pivot = pivots[r];
        const uint64_t flip = (pivot + (n - index)) % n;
        const uint64_t pos = index > flip ? index : flip;
        const uint8_t byte = sources[32ull * ((uint64_t)r * n_blocks + (pos >> 8)) + ((pos & 0xff) >> 3)];
        if ((byte >> (pos & 7)) & 1) index = flip;
    }
    // backwards (the spec's usual direction): out[i] = in[csi(i)];  forwards: out[csi(i)] = in[i]
    if (forwards) out[index] = in[i];
    else out[i] = in[index];
}

// ---------------------------------------------------------------------------------------------
// Committees, proposers and the next sync committee from a resident BeaconState (lhb200_state_committee_cache,
// lhb200_state_beacon_proposer_indices, lhb200_state_next_sync_committee_indices): CommitteeCache::initialized
// (committee_cache.rs:64-125), compute_proposer_index (beacon_state.rs:890-936) and get_next_sync_committee_indices
// (:1091-1125).  The inputs are the handle's own device bytes: its 121-byte validator records and randao_mixes.
constexpr uint32_t SHUFFLE_ROUND_COUNT = 90;
constexpr uint64_t MAX_EFFECTIVE_BALANCE = 32000000000ull, MAX_RANDOM_BYTE = 255;
constexpr uint32_t VAL_EFFECTIVE_BALANCE = 80, VAL_ACTIVATION_EPOCH = 97, VAL_EXIT_EPOCH = 105;

// SHA-256 of a message of at most 55 bytes, given as its one padded block of big-endian words (w is clobbered)
__device__ __forceinline__ void sha256_one_block(uint32_t w[16], uint32_t st[8]) {
    sha256_init(st);
    sha256_compress(st, w);
}
// byte k (0..31) of a digest in word form: a tree of selects on the bits of k >> 2, so that no register array is
// indexed at run time (which would put the digest in local memory)
__device__ __forceinline__ uint32_t digest_byte(const uint32_t st[8], uint32_t k) {
    const bool b0 = k & 4, b1 = k & 8, b2 = k & 16;
    const uint32_t a0 = b0 ? st[1] : st[0], a1 = b0 ? st[3] : st[2], a2 = b0 ? st[5] : st[4], a3 = b0 ? st[7] : st[6];
    const uint32_t w = b2 ? (b1 ? a3 : a2) : (b1 ? a1 : a0);
    return (w >> (24 - 8 * (k & 3))) & 0xff;
}
// little-endian u64 at any byte address: funnel shifts over the three aligned words that cover it (the record fields
// read here end at least 3 bytes before their record does, so no read leaves the record)
__device__ __forceinline__ uint64_t le64_at(const uint8_t* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const uint32_t sh = 8 * (uint32_t)(a & 3), w0 = q[0], w1 = q[1], w2 = q[2];
    return (uint64_t)__funnelshift_r(w0, w1, sh) | ((uint64_t)__funnelshift_r(w1, w2, sh) << 32);
}
// Validator::is_active_at (validator.rs:39-41)
__device__ __forceinline__ bool validator_active_at(const uint8_t* v, uint64_t epoch) {
    return le64_at(v + VAL_ACTIVATION_EPOCH) <= epoch && epoch < le64_at(v + VAL_EXIT_EPOCH);
}

// Ordered active-index compaction (get_active_validator_indices, committee_cache.rs:356-373) in two passes over tiles
// of ACTIVE_TILE records: k_active_count counts each tile's active validators, k_active_write adds up the counts of the
// tiles before its own and writes its tile's indices in ascending order, one 256-record step at a time (a warp ballot
// and the warp counts give each active record its slot).  Both read records at one thread per record, so a warp's
// loads cover 32 consecutive records.
constexpr int ACTIVE_THREADS = 256, ACTIVE_STEPS = 16, ACTIVE_TILE = ACTIVE_THREADS * ACTIVE_STEPS;

__global__ void __launch_bounds__(ACTIVE_THREADS) k_active_count(const uint8_t* __restrict__ vals, uint64_t n,
                                                                 uint64_t epoch, uint32_t* __restrict__ tile_counts) {
    const uint64_t first = (uint64_t)blockIdx.x * ACTIVE_TILE;
    uint32_t cnt = 0;
    for (int k = 0; k < ACTIVE_STEPS; k++) {
        const uint64_t i = first + k * ACTIVE_THREADS + threadIdx.x;
        cnt += i < n && validator_active_at(vals + VAL_SSZ * i, epoch);
    }
    __shared__ uint32_t warp_sum[ACTIVE_THREADS / 32];
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < ACTIVE_THREADS / 32; w++) t += warp_sum[w];
        tile_counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(ACTIVE_THREADS) k_active_write(const uint8_t* __restrict__ vals, uint64_t n,
                                                                 uint64_t epoch, const uint32_t* __restrict__ tile_counts,
                                                                 uint64_t* __restrict__ active,
                                                                 uint64_t* __restrict__ n_active) {
    __shared__ uint64_t warp_sum64[ACTIVE_THREADS / 32];
    __shared__ uint32_t warp_cnt[ACTIVE_THREADS / 32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // this tile's first slot: the active validators of the tiles before it
    uint64_t before = 0;
    for (uint32_t t = threadIdx.x; t < blockIdx.x; t += ACTIVE_THREADS) before += tile_counts[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
    if (lane == 0) warp_sum64[warp] = before;
    __syncthreads();
    uint64_t slot = 0;
#pragma unroll
    for (int w = 0; w < ACTIVE_THREADS / 32; w++) slot += warp_sum64[w];
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *n_active = slot + tile_counts[blockIdx.x];
    const uint64_t first = (uint64_t)blockIdx.x * ACTIVE_TILE;
    for (int k = 0; k < ACTIVE_STEPS; k++) {
        const uint64_t i = first + k * ACTIVE_THREADS + threadIdx.x;
        const bool a = i < n && validator_active_at(vals + VAL_SSZ * i, epoch);
        const uint32_t ballot = __ballot_sync(0xffffffffu, a);
        if (lane == 0) warp_cnt[warp] = __popc(ballot);
        __syncthreads();
        uint64_t at = slot + __popc(ballot & ((1u << lane) - 1));
        uint32_t step = 0;
#pragma unroll
        for (int w = 0; w < ACTIVE_THREADS / 32; w++) {
            at += (uint32_t)w < warp ? warp_cnt[w] : 0;
            step += warp_cnt[w];
        }
        if (a) active[at] = i;
        slot += step;
        __syncthreads();   // warp_cnt is rewritten by the next step
    }
}

// get_seed (beacon_state.rs:1507-1536): H(le32(domain) || le64(epoch) || randao_mixes[(epoch + 65536 - 2) mod 65536]);
// with_slot: the proposer seed of `slot`, H(get_seed(epoch, DOMAIN_BEACON_PROPOSER) || le64(slot)) (:1040-1050).  One
// thread per requested seed.
struct SeedReq {
    uint64_t epoch, slot;
    uint32_t domain, with_slot;
};
constexpr int MAX_SEED_REQS = 32;
struct SeedTable {
    uint32_t n;
    SeedReq r[MAX_SEED_REQS];
};
__global__ void __launch_bounds__(MAX_SEED_REQS) k_committee_seeds(const uint8_t* __restrict__ mixes,
                                                                   const __grid_constant__ SeedTable tab,
                                                                   uint8_t* __restrict__ seeds) {
    if (threadIdx.x >= tab.n) return;
    const SeedReq q = tab.r[threadIdx.x];
    uint32_t w[16], st[8], mix[8];
    load_chunk(mixes + 32 * ((q.epoch % 65536 + 65534) % 65536), mix);
    w[0] = bswap32(q.domain);
    w[1] = bswap32((uint32_t)q.epoch);
    w[2] = bswap32((uint32_t)(q.epoch >> 32));
#pragma unroll
    for (int k = 0; k < 8; k++) w[3 + k] = mix[k];
    w[11] = 0x80000000u;
    w[12] = w[13] = w[14] = 0;
    w[15] = 44 * 8;
    sha256_one_block(w, st);
    if (q.with_slot) {
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = st[k];
        w[8] = bswap32((uint32_t)q.slot);
        w[9] = bswap32((uint32_t)(q.slot >> 32));
        w[10] = 0x80000000u;
        w[11] = w[12] = w[13] = w[14] = 0;
        w[15] = 40 * 8;
        sha256_one_block(w, st);
    }
    store_chunk(seeds + 32 * threadIdx.x, st);
}

// shuffling_positions (committee_cache.rs:110-114): positions[shuffling[i]] = i + 1 over a zero-filled array
__global__ void __launch_bounds__(256) k_shuffling_positions(const uint64_t* __restrict__ shuffling, uint64_t n,
                                                             uint32_t* __restrict__ positions) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) positions[shuffling[i]] = (uint32_t)(i + 1);
}

// Balance-weighted sampling over the active set: candidate i is active[compute_shuffled_index(i mod n, n, seed, 90)],
// accepted when effective_balance * 255 >= MAX_EFFECTIVE_BALANCE * H(seed || le64(i / 32))[i mod 32]; the first `want`
// accepted candidates in order are the seed's winners.  One CTA per seed (the proposer draw: 32 seeds, 1 winner each;
// the sync draw: 1 seed, 512 winners).  The seed's 90 pivots are hashed once into shared memory; then each thread
// takes one speculative candidate of a batch of SAMPLE_THREADS (its 90 source hashes, its record's effective balance,
// its random byte), a ballot and the warp counts order the accepted ones, and batches repeat until the seed has its
// winners.  n <= 2^24 (the host refuses more), so positions and pivots fit 32 bits.
constexpr int SAMPLE_THREADS = 256;
__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample_validators(const uint8_t* __restrict__ seeds,
                                                                      const uint64_t* __restrict__ active, uint32_t n,
                                                                      const uint8_t* __restrict__ vals, uint32_t want,
                                                                      uint64_t* __restrict__ out) {
    __shared__ uint32_t s_seed[8];
    __shared__ uint32_t s_pivot[SHUFFLE_ROUND_COUNT];
    __shared__ uint32_t warp_cnt[SAMPLE_THREADS / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 8) s_seed[tid] = be_word(seeds + 32 * blockIdx.x + 4 * tid);
    __syncthreads();
    uint32_t w[16], st[8];
    if (tid < SHUFFLE_ROUND_COUNT) {   // pivot = le64(H(seed || round)[0:8]) mod n
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = s_seed[k];
        w[8] = (tid << 24) | 0x800000u;
#pragma unroll
        for (int k = 9; k < 15; k++) w[k] = 0;
        w[15] = 33 * 8;
        sha256_one_block(w, st);
        s_pivot[tid] = (uint32_t)((((uint64_t)bswap32(st[1]) << 32) | bswap32(st[0])) % n);
    }
    __syncthreads();
    uint64_t* dst = out + (uint64_t)blockIdx.x * want;
    uint32_t have = 0;
    for (uint64_t base = 0; have < want; base += SAMPLE_THREADS) {
        const uint64_t i = base + tid;
        uint32_t index = (uint32_t)(i % n);
        for (uint32_t r = 0; r < SHUFFLE_ROUND_COUNT; r++) {   // compute_shuffled_index (shuffle_list.rs:18-44)
            uint32_t flip = s_pivot[r] + n - index;
            if (flip >= n) flip -= n;
            const uint32_t pos = index > flip ? index : flip, blk = pos >> 8;
#pragma unroll
            for (int k = 0; k < 8; k++) w[k] = s_seed[k];
            w[8] = (r << 24) | ((blk & 0xff) << 16) | (((blk >> 8) & 0xff) << 8) | ((blk >> 16) & 0xff);
            w[9] = ((blk >> 24) << 24) | 0x800000u;
#pragma unroll
            for (int k = 10; k < 15; k++) w[k] = 0;
            w[15] = 37 * 8;
            sha256_one_block(w, st);
            if ((digest_byte(st, (pos & 0xff) >> 3) >> (pos & 7)) & 1) index = flip;
        }
        const uint64_t cand = active[index];
        const uint64_t eb = le64_at(vals + VAL_SSZ * cand + VAL_EFFECTIVE_BALANCE);
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = s_seed[k];
        w[8] = bswap32((uint32_t)(i >> 5));
        w[9] = bswap32((uint32_t)(i >> 37));
        w[10] = 0x80000000u;
#pragma unroll
        for (int k = 11; k < 15; k++) w[k] = 0;
        w[15] = 40 * 8;
        sha256_one_block(w, st);
        const bool ok = eb * MAX_RANDOM_BYTE >= MAX_EFFECTIVE_BALANCE * digest_byte(st, (uint32_t)(i & 31));
        const uint32_t ballot = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) warp_cnt[warp] = __popc(ballot);
        __syncthreads();
        uint32_t at = have + __popc(ballot & ((1u << lane) - 1)), step = 0;
#pragma unroll
        for (int k = 0; k < SAMPLE_THREADS / 32; k++) {
            at += (uint32_t)k < warp ? warp_cnt[k] : 0;
            step += warp_cnt[k];
        }
        if (ok && at < want) dst[at] = cand;
        have += step;
        __syncthreads();   // warp_cnt is rewritten by the next batch
    }
}

}  // namespace lhb200
