// merkle_host.cu — host driver + C ABI of the tree-hash path.
//
// Host code only plans (offset parsing, literal chunk packing, launch tables); every SHA-256 compression
// runs on the device.  Mirrors, at the batch level, tree_hash::{merkle_root, mix_in_length, MerkleHasher},
// merkle_proof::MerkleTree and BeaconState::update_tree_hash_cache (cold) — see include/lhb200.h.
#include <string.h>
#include <algorithm>
#include <array>
#include <memory>
#include <type_traits>
#include <unordered_map>
#include <vector>
#include "ctx.h"
#include "merkle.cuh"

namespace lhb200 {

static inline uint64_t ceil_div(uint64_t a, uint64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline uint32_t ceil_log2(uint64_t x) {
    uint32_t d = 0;
    while ((1ull << d) < x) d++;
    return d;
}

int32_t merkle_init() {
    Ctx& c = ctx();
    k_init_zero_hashes<<<1, 32, 0, c.stream>>>();
    count_launch();
    LHB_CUDA(cudaGetLastError());
    uint32_t words[MAX_ZERO_DEPTH + 1][8];
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    LHB_CUDA(cudaMemcpyFromSymbol(words, g_zero_words, sizeof words));
    for (int d = 0; d <= MAX_ZERO_DEPTH; d++)
        for (int i = 0; i < 8; i++) {
            c.zero_hashes[d][4 * i + 0] = words[d][i] >> 24;
            c.zero_hashes[d][4 * i + 1] = words[d][i] >> 16;
            c.zero_hashes[d][4 * i + 2] = words[d][i] >> 8;
            c.zero_hashes[d][4 * i + 3] = words[d][i];
        }
    return LHB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Plan: everything needed to hash one object — leaf kernels, reduce passes, the tail hash program.
// All device memory a plan touches lives in one arena: [staged inputs | scratch nodes | literals | slots].

// The leaf kernel of a big list turns each fixed-size SSZ item into its 32-byte root, at `units` hash32_concat each.
// `tree` is the TreeDev kind that recomputes one leaf on the warm path.
struct LeafKind {
    enum Kernel { NONE, VALIDATORS, RECORDS, HASH_PAIRS } kernel;   // NONE: the items already are the chunks
    uint32_t tree;                                                  // RECORDS: TREE_RECORDS + its k_record_roots kind
    uint32_t units;
};
constexpr LeafKind LEAF_NONE{LeafKind::NONE, TREE_CHUNKS, 0},
                   LEAF_VALIDATOR{LeafKind::VALIDATORS, TREE_VALIDATORS, 8},
                   LEAF_PUBKEY{LeafKind::RECORDS, TREE_RECORDS + REC_PUBKEY, 1},
                   LEAF_ETH1_DATA{LeafKind::RECORDS, TREE_RECORDS + REC_ETH1_DATA, 3},
                   LEAF_U64_PAIR{LeafKind::RECORDS, TREE_RECORDS + REC_U64_PAIR, 1},
                   LEAF_U64_TRIPLE{LeafKind::RECORDS, TREE_RECORDS + REC_U64_TRIPLE, 3},
                   LEAF_DEPOSIT_REQUEST{LeafKind::RECORDS, TREE_RECORDS + REC_DEPOSIT_REQUEST, 10},
                   // HistoricalSummary {H256, H256}: one pair hash, which the warm path runs as a record
                   LEAF_CHUNK_PAIR{LeafKind::HASH_PAIRS, TREE_RECORDS + REC_HISTORICAL_SUMMARY, 1};

struct LeafLaunch {
    LeafKind kind;
    const uint8_t* in;
    uint8_t* out;
    uint64_t n;
};

struct Plan {
    uint8_t* arena = nullptr;   // device base
    size_t arena_bytes = 0;
    size_t bump = 0;            // allocation cursor (bytes)
    std::vector<uint8_t> lit;   // host literal block (32-byte chunks), copied to arena+lit_off
    size_t lit_off = 0, lit_cap = 0;
    std::vector<LeafLaunch> leaves;
    std::vector<std::vector<MerkleSeg>> passes;
    std::vector<HashOp> ops;
    std::vector<int> op_wave;
    // op outputs come from a dense node pool right after the literals, so "which wave produces this operand" is an
    // array lookup (a slot table over the whole 72 MB state arena made every plan build slow)
    size_t node_off = 0, node_cap = 0, node_used = 0;
    bool node_overflow = false;
    std::vector<int16_t> slot_wave;                    // pool slot -> wave producing it
    uint64_t forced_base = 0;                          // forced destinations (block batch outputs): one dense range
    std::vector<int16_t> forced_wave;
    std::vector<ByteItem> items;                       // packed byte strings hashed straight from the staged blob
    ByteItem* d_items = nullptr;
    std::vector<int32_t> h_waves;                      // host copy of the wave table (wide waves get their own launch)
    uint64_t forced_dst = 0;                           // destination of the next op_hash (0 = allocate)
    // big fields of a staged state that keep a tree for the warm path (lhb200_state_enable_incremental): where their
    // leaf chunks live, where the tail program reads their data root, and the staged copy (SSZ items) they come from
    struct TreeSpec { const uint8_t* chunks; uint64_t n_chunks; uint64_t top_addr; const uint8_t* src; LeafKind leaf;
                      size_t copy; uint32_t item_bytes; };
    std::vector<TreeSpec> trees;
    // every merkle_list folded by reduce passes: its leaf chunks and the address of its data root at level
    // ceil_log2(n), where a Merkle proof that enters the list rebuilds its levels (lhb200_state_proofs)
    struct ListRec { const uint8_t* chunks; uint64_t n; uint64_t top_addr; };
    std::vector<ListRec> merkle_lists;
    uint64_t hash_units = 0;
    // SSZ provenance of literal chunks (for lhb200_state_patch): chunk index <- n bytes at SSZ offset src_off
    struct LitSrc { uint32_t lit_index; uint32_t n; uint64_t src_off; };
    std::vector<LitSrc> lit_src;
    const uint8_t* ssz_base = nullptr;
    uint64_t ssz_len = 0;
    // tail program (device copies)
    HashOp* d_ops = nullptr;
    int32_t* d_waves = nullptr;
    int n_waves = 0;

    uint8_t* alloc(size_t nbytes, size_t align = 256) {  // device sub-allocation
        size_t off = align_up(bump, align);
        bump = off + nbytes;
        return arena ? arena + off : reinterpret_cast<uint8_t*>(off);
    }
    static uint64_t zero_op(uint32_t level) { return OP_ZERO_FLAG | level; }
    uint64_t literal_raw(const uint8_t chunk[32]) {
        size_t i = lit.size();
        lit.resize(i + 32);
        memcpy(&lit[i], chunk, 32);
        return reinterpret_cast<uint64_t>(arena + lit_off + i);
    }
    uint64_t literal_bytes(const uint8_t* p, size_t n) {  // zero-padded chunk from <=32 bytes
        uint8_t c[32] = {0};
        memcpy(c, p, n);
        if (ssz_base && p >= ssz_base && p + n <= ssz_base + ssz_len)
            lit_src.push_back({(uint32_t)(lit.size() / 32), (uint32_t)n, (uint64_t)(p - ssz_base)});
        return literal_raw(c);
    }
    uint64_t literal_u64(uint64_t v) {
        uint8_t c[32] = {0};
        for (int k = 0; k < 8; k++) c[k] = (uint8_t)(v >> (8 * k));
        return literal_raw(c);
    }
    int wave_of(uint64_t operand) const {
        if (operand & OP_ZERO_FLAG) return -1;
        const size_t slot = (operand - reinterpret_cast<uint64_t>(arena) - node_off) / 32;  // outside the pool: huge
        if (slot < slot_wave.size()) return slot_wave[slot];
        const size_t fs = (operand - forced_base) / 32;
        if (fs < forced_wave.size()) return forced_wave[fs];
        return -1;  // staged data / literals / leaf outputs: ready at start
    }
    uint64_t op_hash(uint64_t a, uint64_t b) {
        const int w = std::max(wave_of(a), wave_of(b)) + 1;
        uint64_t dst;
        if (forced_dst) {
            dst = forced_dst;
            forced_dst = 0;
            const size_t fs = (dst - forced_base) / 32;
            if (fs < forced_wave.size()) forced_wave[fs] = (int16_t)w;
        } else {
            if (node_used >= node_cap) { node_overflow = true; node_used = 0; }  // reported by build_plan
            dst = reinterpret_cast<uint64_t>(arena) + node_off + 32 * node_used;
            if (node_used >= slot_wave.size()) slot_wave.resize(std::max<size_t>(node_used + 1, 2 * slot_wave.size()), -1);
            slot_wave[node_used++] = (int16_t)w;
        }
        ops.push_back({dst, a, b});
        op_wave.push_back(w);
        hash_units++;
        return dst;
    }
    uint64_t mix_in_length(uint64_t root, uint64_t len) { return op_hash(root, literal_u64(len)); }
    // merkleize k operands over next_pow2(k) leaves (container / small vectors), padding with zero hashes
    // `final_dst` (optional): device address that receives the root (depth >= 1)
    uint64_t small_tree(std::vector<uint64_t> nodes, uint32_t depth, uint64_t final_dst = 0) {
        if (nodes.empty()) return zero_op(depth);
        for (uint32_t l = 0; l < depth; l++) {
            std::vector<uint64_t> nx;
            for (size_t i = 0; i < nodes.size(); i += 2) {
                if (l + 1 == depth) forced_dst = final_dst;
                nx.push_back(op_hash(nodes[i], i + 1 < nodes.size() ? nodes[i + 1] : zero_op(l)));
            }
            nodes.swap(nx);
        }
        return nodes[0];
    }
    uint64_t container(const std::vector<uint64_t>& fields, uint64_t final_dst = 0) {
        return small_tree(fields, ceil_log2(fields.size()), final_dst);
    }
    // hash_tree_root of a packed byte string resident at d_src (any alignment): merkleize(pack(bytes), 2^depth),
    // optionally mixed in with `length`; `last_mask` is ANDed onto the last byte (bitlist delimiter removal)
    uint64_t bytes_item(const uint8_t* d_src, uint64_t nbytes, uint32_t depth, bool mix, uint64_t length = 0,
                        uint32_t last_mask = 0xff) {
        uint8_t* out = alloc(32, 32);
        ByteItem it;
        it.src = d_src; it.nbytes = nbytes; it.out = out; it.length = length; it.depth = depth;
        it.flags = (mix ? 1u : 0u) | (last_mask << 8);
        items.push_back(it);
        uint64_t n = (nbytes + 31) / 32;
        for (uint32_t l = 1; l <= depth && n > 1; l++) { n = (n + 1) / 2; hash_units += n; }
        hash_units += mix ? 1 : 0;
        return reinterpret_cast<uint64_t>(out);
    }
    // merkleize n chunks resident at d_in (16-B aligned) with limit 2^depth.  `warm` (optional: src, leaf, copy and
    // item_bytes) is recorded in `trees` with the chunks and the data root when reduce passes build the tree.
    uint64_t merkle_list(const uint8_t* d_in, uint64_t n, uint32_t depth, const TreeSpec* warm = nullptr) {
        if (n == 0) return zero_op(depth);
        if (n <= 8) {
            std::vector<uint64_t> nodes;
            for (uint64_t i = 0; i < n; i++) nodes.push_back(reinterpret_cast<uint64_t>(d_in + 32 * i));
            uint32_t d0 = std::min(depth, ceil_log2(n));
            uint64_t r = small_tree(nodes, d0);
            for (uint32_t l = d0; l < depth; l++) r = op_hash(r, zero_op(l));
            return r;
        }
        uint32_t level = 0;
        const uint8_t* in = d_in;
        size_t p = 0;
        const uint64_t hash_units_n0 = n;  // leaf count of this list
        while (n > 1 && level < depth) {
            uint32_t tl = std::min<uint32_t>(MAX_TILE_LOG, depth - level);
            tl = std::min<uint32_t>(tl, ceil_log2(n));  // do not fold past the single-root level here
            uint64_t n_out = ceil_div(n, 1ull << tl);
            uint8_t* out = alloc(n_out * 32);
            if (passes.size() <= p) passes.resize(p + 1);
            MerkleSeg sg;
            sg.in = in; sg.out = out; sg.n_in = n; sg.level_in = level; sg.tile_log = tl;
            sg.cta_begin = 0; sg.n_tiles = (uint32_t)n_out;
            passes[p++].push_back(sg);
            // hashes actually performed: nodes with a valid left child at each level
            for (uint32_t l = 1; l <= tl; l++) hash_units += ceil_div(n, 1ull << l);
            level += tl;
            n = n_out;
            in = out;
        }
        uint64_t r = reinterpret_cast<uint64_t>(in);
        merkle_lists.push_back({d_in, hash_units_n0, r});
        if (warm) trees.push_back({d_in, hash_units_n0, r, warm->src, warm->leaf, warm->copy, warm->item_bytes});
        for (uint32_t l = level; l < depth; l++) r = op_hash(r, zero_op(l));
        return r;
    }
    uint8_t* leaf_kernel(LeafKind kind, const uint8_t* in, uint64_t n) {
        uint8_t* out = alloc(std::max<uint64_t>(n, 1) * 32);
        if (n) leaves.push_back({kind, in, out, n});
        hash_units += (uint64_t)kind.units * n;
        return out;
    }
};

static int32_t plan_enqueue_tail(Plan& pl, cudaStream_t s);
// Roots of n validators (TREE_VALIDATORS) or records (TREE_RECORDS + kind) at `in` -> chunks at `out`.  e0 / e1
// (optional) are recorded around k_validator_roots.
static void enqueue_leaf_roots(uint32_t tree_kind, const uint8_t* in, uint64_t n, uint8_t* out, cudaStream_t s,
                               cudaEvent_t e0, cudaEvent_t e1) {
    if (tree_kind == TREE_VALIDATORS) {
        if (e0) cudaEventRecord(e0, s);
        k_validator_roots<<<(unsigned)ceil_div(n, VAL_PER_CTA), VAL_PER_CTA, 0, s>>>(in, n, out);
        if (e1) cudaEventRecord(e1, s);
    } else {
        k_record_roots<<<(unsigned)ceil_div(n, 128), 128, 0, s>>>(in, n, (int)(tree_kind - TREE_RECORDS), out);
    }
    count_launch();
}
// Leaf kernels, reduce passes and byte items of a plan: everything before its tail hash program.
static void plan_enqueue_body(Plan& pl, cudaStream_t s, cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr) {
    for (const LeafLaunch& L : pl.leaves) {   // leaf_kernel is never called without a kernel
        if (L.kind.kernel == LeafKind::HASH_PAIRS) {
            k_hash_pairs<<<(unsigned)ceil_div(L.n, 256), 256, 0, s>>>(L.in, L.out, L.n);
            count_launch();
        } else {
            enqueue_leaf_roots(L.kind.tree, L.in, L.n, L.out, s, e0, e1);
        }
    }
    for (auto& pass : pl.passes) {
        for (size_t i = 0; i < pass.size(); i += MAX_SEGS) {
            MerkleSegTable tab;
            tab.n = (int)std::min<size_t>(MAX_SEGS, pass.size() - i);
            uint32_t ctas = 0;
            for (int k = 0; k < tab.n; k++) {
                tab.s[k] = pass[i + k];
                tab.s[k].cta_begin = ctas;
                ctas += tab.s[k].n_tiles;
            }
            k_merkle_reduce<<<ctas, REDUCE_THREADS, 0, s>>>(tab);
            count_launch();
        }
    }
    if (!pl.items.empty()) {
        k_byte_items<<<(unsigned)pl.items.size(), ITEM_THREADS, 0, s>>>(pl.d_items);
        count_launch();
    }
}
// Enqueue a finished plan on `s`.  Literals must already be in the arena.
static int32_t plan_enqueue(Plan& pl, cudaStream_t s, cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr) {
    plan_enqueue_body(pl, s, e0, e1);
    return plan_enqueue_tail(pl, s);
}
// The tail hash program only (zero ladders, length mix-ins, containers): all a warm root needs after the trees.
static int32_t plan_enqueue_tail(Plan& pl, cudaStream_t s) {
    // narrow waves run back to back inside one CTA; a wide wave (block batches) gets the whole grid
    constexpr int WIDE_WAVE = 1024;
    for (int w = 0; w < pl.n_waves;) {
        const int cnt = pl.h_waves[w + 1] - pl.h_waves[w];
        if (cnt >= WIDE_WAVE) {
            k_hash_ops<<<(unsigned)ceil_div(cnt, PROG_THREADS), PROG_THREADS, 0, s>>>(pl.d_ops + pl.h_waves[w], cnt);
            w++;
        } else {
            int e = w;
            while (e < pl.n_waves && pl.h_waves[e + 1] - pl.h_waves[e] < WIDE_WAVE) e++;
            k_hash_program<<<1, PROG_THREADS, 0, s>>>(pl.d_ops, pl.d_waves + w, e - w);
            w = e;
        }
        count_launch();
    }
    LHB_CUDA(cudaGetLastError());
    return LHB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Plan lifecycle: size, take an arena, build, upload literals and program, enqueue, read the root.

// Device bytes of the program blobs plan_upload allocates from the arena: ops, wave table (at most one entry per op,
// plus one) and byte items, each 256-byte aligned.
static size_t program_bytes(size_t n_ops, size_t n_items) {
    return align_up(n_ops * sizeof(HashOp), 256) + align_up((n_ops + 2) * 4, 256) +
           align_up(n_items * sizeof(ByteItem), 256) + 512;
}
// Pinned staging plan_upload needs: literals, then the program blobs.
static size_t plan_stage_bytes(const Plan& pl) {
    return align_up(pl.lit.size(), 256) + program_bytes(pl.ops.size(), pl.items.size());
}

// Run `build` over the arena (null: a dry run that only sizes).  `build` must be deterministic in its allocation
// sequence and returns a status.
template <class F>
static int32_t build_plan(Plan& pl, uint8_t* arena, size_t arena_bytes, size_t lit_cap, F&& build,
                          size_t node_cap = 8192) {
    pl = Plan();
    pl.arena = arena;
    pl.arena_bytes = arena_bytes;
    pl.lit_cap = lit_cap;
    pl.lit_off = 0;
    pl.node_off = align_up(lit_cap, 256);   // literals first, then the node pool
    pl.node_cap = node_cap;
    pl.bump = pl.node_off + node_cap * 32;
    const int32_t rc = build(pl);
    if (rc) return rc;
    if (pl.lit.size() > lit_cap) {
        set_error("internal: literal block overflow (%zu > %zu)", pl.lit.size(), lit_cap);
        return LHB200_EINVAL;
    }
    if (pl.node_overflow) {
        set_error("internal: hash program larger than its node pool (%zu nodes)", node_cap);
        return LHB200_EINVAL;
    }
    return LHB200_OK;
}

// Size-then-build: a dry run over a null arena gives the plan's footprint; take(need, &arena, &bytes) supplies an
// arena of bytes >= need (the build, its program blobs and `extra` bytes the caller allocates after the build), and
// the build runs again over it.
template <class F, class T>
static int32_t build_sized(Plan& pl, size_t lit_cap, size_t extra, F&& build, T&& take) {
    Plan dry;
    int32_t rc = build_plan(dry, nullptr, 0, lit_cap, build);
    if (rc) return rc;
    uint8_t* arena = nullptr;
    size_t bytes = 0;
    rc = take(align_up(dry.bump, 256) + program_bytes(dry.ops.size(), dry.items.size()) + extra, &arena, &bytes);
    if (rc) return rc;
    return build_plan(pl, arena, bytes, lit_cap, build);
}
static int32_t scratch_arena(size_t need, uint8_t** arena, size_t* bytes) {
    *arena = static_cast<uint8_t*>(dev_scratch(need));
    *bytes = need;
    return *arena ? LHB200_OK : LHB200_ENOMEM;
}

// The wave table of a plan's ops (h_waves[w]: first op of wave w) and the ops in wave order at h_ops (stable
// counting sort).
static void plan_sort_ops(Plan& pl, HashOp* h_ops) {
    int nw = 0;
    for (int w : pl.op_wave) nw = std::max(nw, w + 1);
    pl.n_waves = nw;
    pl.h_waves.assign(nw + 1, 0);
    for (int w : pl.op_wave) pl.h_waves[w + 1]++;
    for (int w = 0; w < nw; w++) pl.h_waves[w + 1] += pl.h_waves[w];
    std::vector<int32_t> next(pl.h_waves.begin(), pl.h_waves.end() - 1);
    for (size_t i = 0; i < pl.ops.size(); i++) h_ops[next[pl.op_wave[i]]++] = pl.ops[i];
}

// Sort the ops by wave and upload literals and program (ops, wave table, byte items) through the pinned `h_stage`
// (plan_stage_bytes).  The program blobs are allocated from the arena after everything else the plan holds; a plan
// they would not fit is refused before any copy.
static int32_t plan_upload(Plan& pl, cudaStream_t s, uint8_t* h_stage) {
    const size_t prog = program_bytes(pl.ops.size(), pl.items.size());
    if (pl.bump + prog > pl.arena_bytes) {
        set_error("internal: plan exceeds its arena (%zu + %zu program bytes of %zu)", pl.bump, prog, pl.arena_bytes);
        return LHB200_EINVAL;
    }
    uint8_t* h = h_stage;
    if (!pl.lit.empty()) {
        memcpy(h, pl.lit.data(), pl.lit.size());
        LHB_CUDA(cudaMemcpyAsync(pl.arena + pl.lit_off, h, pl.lit.size(), cudaMemcpyHostToDevice, s));
        h += align_up(pl.lit.size(), 256);
    }
    plan_sort_ops(pl, reinterpret_cast<HashOp*>(h));
    if (!pl.ops.empty()) {
        const size_t nb = pl.ops.size() * sizeof(HashOp), wb = pl.h_waves.size() * sizeof(int32_t);
        pl.d_ops = reinterpret_cast<HashOp*>(pl.alloc(nb));
        LHB_CUDA(cudaMemcpyAsync(pl.d_ops, h, nb, cudaMemcpyHostToDevice, s));
        h += align_up(nb, 256);
        memcpy(h, pl.h_waves.data(), wb);
        pl.d_waves = reinterpret_cast<int32_t*>(pl.alloc(wb));
        LHB_CUDA(cudaMemcpyAsync(pl.d_waves, h, wb, cudaMemcpyHostToDevice, s));
        h += align_up(wb, 256);
    }
    if (!pl.items.empty()) {
        const size_t ib = pl.items.size() * sizeof(ByteItem);
        memcpy(h, pl.items.data(), ib);
        pl.d_items = reinterpret_cast<ByteItem*>(pl.alloc(ib));
        LHB_CUDA(cudaMemcpyAsync(pl.d_items, h, ib, cudaMemcpyHostToDevice, s));
    }
    return LHB200_OK;
}

// Host input of H2D copies.  Pinned host memory (and device memory) is read by the copy engine directly; pageable
// memory is first bounced through the pinned slab, which then needs bounce_bytes() for it.
struct HostInput {
    const uint8_t* p;
    size_t n;
    bool direct;
    HostInput(const uint8_t* p_, size_t n_, bool on_device = false) : p(p_), n(n_), direct(on_device || !n) {
        cudaPointerAttributes at;
        if (!direct) direct = cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost;
        cudaGetLastError();
    }
    size_t bounce_bytes() const { return direct ? 0 : align_up(n, 256); }
    const uint8_t* source(uint8_t* slab) const { return direct ? p : static_cast<const uint8_t*>(memcpy(slab, p, n)); }
};

// Copy a root operand to `dst` on s.  A zero-hash constant has no device address: it comes from the host table,
// through the pinned `h32` (which may be `dst` itself).
static int32_t read_root(uint64_t root, void* dst, cudaMemcpyKind kind, uint8_t* h32, cudaStream_t s) {
    if (!(root & OP_ZERO_FLAG)) {
        LHB_CUDA(cudaMemcpyAsync(dst, reinterpret_cast<const void*>(root), 32, kind, s));
        return LHB200_OK;
    }
    memcpy(h32, ctx().zero_hashes[root & 0xff], 32);
    if (dst != h32) LHB_CUDA(cudaMemcpyAsync(dst, h32, 32, cudaMemcpyHostToDevice, s));
    return LHB200_OK;
}

// Generic runner for "one input blob -> one root" host entry points.
//   describe(plan, d_in) describes the work given the device copy of the input and returns the root operand.
template <class F>
static int32_t run_simple(const uint8_t* h_in, size_t in_bytes, uint8_t out[32], F&& describe, bool in_on_device = false) {
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const size_t in_pad = align_up(in_bytes + 32, 256);
    uint64_t root = 0;
    uint8_t* d_in = nullptr;
    Plan pl;
    int32_t rc = build_sized(pl, 4096, 256, [&](Plan& p) {
        d_in = p.alloc(in_pad);
        root = describe(p, d_in);
        return LHB200_OK;
    }, scratch_arena);
    if (rc) return rc;
    const HostInput in(h_in, in_bytes, in_on_device);
    const size_t ho = in.bounce_bytes(), hr = ho + align_up(plan_stage_bytes(pl), 256);
    uint8_t* hst = static_cast<uint8_t*>(pinned_scratch(hr + 32));
    if (!hst) return LHB200_ENOMEM;
    // H2D input (zero the padding tail so packed lists see zero-filled last chunks)
    LHB_CUDA(cudaMemsetAsync(d_in + in_bytes / 256 * 256, 0, in_pad - in_bytes / 256 * 256, c.stream));
    if (in_bytes) LHB_CUDA(cudaMemcpyAsync(d_in, in.source(hst), in_bytes, cudaMemcpyDefault, c.stream));
    rc = plan_upload(pl, c.stream, hst + ho);
    if (rc) return rc;
    rc = plan_enqueue(pl, c.stream);
    if (rc) return rc;
    rc = read_root(root, hst + hr, cudaMemcpyDeviceToHost, hst + hr, c.stream);
    if (rc) return rc;
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out, hst + hr, 32);
    return LHB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// SSZ layouts (mainnet preset).  Forks only append fields to a container, so every field sits at the same offset in
// each fork that has it: the positions below hold for all forks, and a fork's row in FORK_LAYOUTS says how many of
// the fields it has, how large the fixed parts are and which limits apply.
namespace state_layout {
constexpr uint32_t O_GENESIS_TIME = 0, O_GVR = 8, O_SLOT = 40, O_FORK = 48, O_LBH = 64, O_BLOCK_ROOTS = 176,
                   O_STATE_ROOTS = 262320, O_HIST_OFF = 524464, O_ETH1_DATA = 524468, O_VOTES_OFF = 524540,
                   O_DEPOSIT_INDEX = 524544, O_VAL_OFF = 524552, O_BAL_OFF = 524556, O_RANDAO = 524560,
                   O_SLASHINGS = 2621712, O_PP_OFF = 2687248, O_CP_OFF = 2687252, O_JUST = 2687256,
                   O_PJC = 2687257, O_CJC = 2687297, O_FC = 2687337, O_INACT_OFF = 2687377, O_CSC = 2687381,
                   O_NSC = 2712005, O_LEPH_OFF = 2736629, O_NWI = 2736633, O_NWVI = 2736641, O_HS_OFF = 2736649,
                   O_ELECTRA_U64 = 2736653, O_PBD_OFF = 2736701, O_PPW_OFF = 2736705, O_PC_OFF = 2736709;
constexpr uint32_t SYNC_COMMITTEE_BYTES = 513 * 48;
// offsets of the variable-size fields, in field order
constexpr uint32_t VAR_POS[] = {O_HIST_OFF, O_VOTES_OFF, O_VAL_OFF, O_BAL_OFF, O_PP_OFF, O_CP_OFF, O_INACT_OFF,
                                O_LEPH_OFF, O_HS_OFF, O_PBD_OFF, O_PPW_OFF, O_PC_OFF};
enum { V_HIST, V_VOTES, V_VAL, V_BAL, V_PP, V_CP, V_INACT, V_LEPH, V_HS, V_PBD, V_PPW, V_PC, N_VAR };
}  // namespace state_layout

namespace block_layout {
constexpr uint32_t BLOCK_FIXED = 84, BLOCK_VAR_POS[] = {80};   // body
// BeaconBlockBody: proposer_slashings, attester_slashings, attestations, deposits, voluntary_exits, execution_payload,
// bls_to_execution_changes, blob_kzg_commitments, consolidations
constexpr uint32_t BODY_VAR_POS[] = {200, 204, 208, 212, 216, 380, 384, 388, 392};
enum { B_PROPOSER_SLASHINGS, B_ATTESTER_SLASHINGS, B_ATTESTATIONS, B_DEPOSITS, B_EXITS, B_PAYLOAD, B_BLS_CHANGES,
       B_KZG_COMMITMENTS, B_CONSOLIDATIONS, N_BODY_VAR };
// ExecutionPayload: extra_data, transactions, withdrawals, deposit_requests, withdrawal_requests; the header has the
// same extra_data offset and no other variable-size field
constexpr uint32_t PAYLOAD_VAR_POS[] = {436, 504, 508, 528, 532}, HEADER_VAR_POS[] = {436};
enum { P_EXTRA_DATA, P_TRANSACTIONS, P_WITHDRAWALS, P_DEPOSIT_REQUESTS, P_WITHDRAWAL_REQUESTS, N_PAYLOAD_VAR };
constexpr uint32_t PAYLOAD_PREFIX_FIELDS = 13;   // parent_hash .. block_hash: the same in payload and header
// Attestation and IndexedAttestation: the bit or index list is the first field; AttesterSlashing: two
// IndexedAttestations behind an 8-byte fixed part
constexpr uint32_t FIRST_VAR_POS[] = {0}, ATTESTER_SLASHING_VAR_POS[] = {0, 4};
}  // namespace block_layout

// One row per fork from Altair to Electra (beacon_state.rs:224-571, beacon_block_body.rs:43-121,
// execution_payload.rs:54-101, execution_payload_header.rs:46-93, attestation.rs:76-82; limits eth_spec.rs:389-440).
struct ForkLayout {
    int state_fields, body_fields, payload_fields;   // payload_fields: also the header's; 0 before Bellatrix
    uint32_t state_fixed, header_fixed, body_fixed, payload_fixed, attestation_fixed;
    // Attestation.aggregation_bits, IndexedAttestation.attesting_indices, BeaconBlockBody.{attestations, attester_slashings}
    uint64_t max_aggregation_bits, max_attesting_indices, max_attestations, max_attester_slashings;
};
constexpr ForkLayout FORK_LAYOUTS[] = {
    // fields: state, body, payload   fixed parts: state, header, body, payload, attestation   limits
    {24,  9,  0, 2736629,   0, 380,   0, 228,   2048,   2048, 128, 2},   // Altair
    {25, 10, 14, 2736633, 536, 384, 508, 228,   2048,   2048, 128, 2},   // Bellatrix
    {28, 11, 15, 2736653, 568, 388, 512, 228,   2048,   2048, 128, 2},   // Capella
    {28, 12, 17, 2736653, 584, 392, 528, 228,   2048,   2048, 128, 2},   // Deneb
    {37, 13, 19, 2736713, 648, 396, 536, 236, 131072, 131072,   8, 1},   // Electra
};
static const ForkLayout* fork_layout(int32_t fork) {
    return fork >= LHB200_FORK_ALTAIR && fork <= LHB200_FORK_ELECTRA ? &FORK_LAYOUTS[fork - LHB200_FORK_ALTAIR] : nullptr;
}
constexpr int MAX_FIELDS = FORK_LAYOUTS[LHB200_FORK_ELECTRA - LHB200_FORK_ALTAIR].state_fields;   // the widest state
// chunk-tree depth of a packed list of at most `nbytes` bytes
static inline uint32_t packed_depth(uint64_t nbytes) { return ceil_log2(ceil_div(nbytes, 32)); }

static inline uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// Bytes [off, off + len) of one variable-size field, relative to its container.
struct Span {
    uint64_t off, len;
    // a whole number of `item`-byte items, at most `limit` of them
    bool fits(uint64_t item, uint64_t limit) const { return len % item == 0 && len / item <= limit; }
};
// The variable-size fields of the SSZ container s[0, len) with a `fixed`-byte fixed part: field k's offset is at
// pos[k].  A field whose offset would lie past the fixed part is one this fork does not have (forks only append), is
// not read and gets an empty span at the end.  False unless the first offset is the fixed size, the offsets never
// decrease and the last is at most len.
template <size_t N>
static bool read_offsets(const uint8_t* s, uint64_t len, uint32_t fixed, const uint32_t (&pos)[N], Span (&span)[N]) {
    if (len < fixed) return false;
    uint64_t at[N + 1];
    size_t n = 0;
    for (; n < N && pos[n] + 4 <= fixed; n++) {
        at[n] = rd32(s + pos[n]);
        if (n == 0 ? at[0] != fixed : at[n] < at[n - 1]) return false;
    }
    if (n && at[n - 1] > len) return false;
    for (size_t k = n; k <= N; k++) at[k] = len;
    for (size_t k = 0; k < N; k++) span[k] = {at[k], at[k + 1] - at[k]};
    return true;
}

}  // namespace lhb200

namespace lhb200 {
// Multi-GPU sharding of one state (SURVEY §8e): rank r of `world` (a power of two) owns the leaf range
// [r * 2^s, (r+1) * 2^s) of every big list (s = ceil_log2(#chunks) - log2(world)) and produces the 32-byte root of
// that height-s subtree; small fields are computed by every rank.  After one all-gather of the subtree roots each
// rank folds them (log2(world) levels + zero ladder + length mix-in + the 32-leaf container) in lhb200_state_combine.
struct StageCopy {
    size_t src_off, nbytes;
    uint8_t* dst;
    size_t pad_to;  // zero-fill up to this many bytes at dst
};

// Sizes of a staged state's plan and copies when the describer starts a field: field k emitted everything from
// marks[k] up to marks[k + 1], which is how a conversion to resizable lists drops the lists' share of the plan.
struct PlanMark {
    size_t ops, leaves, copies, trees, merkle_lists;
    std::vector<size_t> passes;   // segments of each reduce pass
    size_t pass(size_t q) const { return q < passes.size() ? passes[q] : 0; }
};

struct ShardCfg {
    uint32_t rank = 0, world = 1;
    int32_t fork = LHB200_FORK_DENEB;   // which BeaconState variant the SSZ is (FORK_LAYOUTS)
};
struct ShardedList {
    int field;            // index in the state container
    uint32_t s;           // height of the per-rank subtree
    uint32_t limit_depth; // chunk-tree depth of the list limit
    uint64_t mix_len;     // length to mix in (lists); UINT64_MAX = vector (no mix-in)
    uint64_t local_op;    // operand holding this rank's subtree root
};

}  // namespace lhb200

static uint8_t* g_spare_arena = nullptr;  // guarded by ctx().mu
static size_t g_spare_bytes = 0;
static cudaEvent_t g_proof_ev[2] = {nullptr, nullptr};   // around the last k_proof_branches launch
// lhb200_shutdown: the recycled arena and the events belong to the context that is going away
namespace lhb200 {
void merkle_shutdown();
}
void lhb200::merkle_shutdown() {
    if (g_spare_arena) cudaFree(g_spare_arena);
    g_spare_arena = nullptr;
    g_spare_bytes = 0;
    for (cudaEvent_t& e : g_proof_ev) {
        if (e) cudaEventDestroy(e);
        e = nullptr;
    }
}

struct lhb200_state {
    uint8_t* arena = nullptr;
    size_t arena_bytes = 0;
    lhb200::Plan plan;
    uint64_t field_ops[lhb200::MAX_FIELDS];
    uint64_t root_op = 0;
    lhb200::HashOp* d_gather = nullptr;   // operand table: root_op, field_ops, then the sharded lists' local_op
    uint8_t* d_result = nullptr;  // (1 + MAX_FIELDS) * 32 bytes: root + field roots gathered
    cudaEvent_t e_k0 = nullptr, e_k1 = nullptr;  // around k_validator_roots
    lhb200::ShardCfg shard;
    std::vector<lhb200::ShardedList> sharded;
    uint8_t* d_coll = nullptr;              // lhb200_state_root_sharded: own subtree roots | all ranks' roots
    std::vector<lhb200::StageCopy> copies;  // SSZ ranges resident in the arena (for lhb200_state_patch)
    std::vector<uint32_t> copy_order, lit_order;   // offset-sorted indices into copies / plan.lit_src (patch lookups)
    std::vector<int32_t> copy_tree;         // copies[k] -> index of its resident tree (warm path), -1 if none
    std::vector<lhb200::PlanMark> marks;    // per field, and one past the last (PlanMark)
    // warm path (lhb200_state_enable_incremental): full level arrays per big list + dirty leaves since the last root
    // dirty leaves since the last root: a host BITMAP per tree (marking is O(1) per edit and dedups for free; the next
    // root extracts the sorted index list with a ctz scan — no sort) plus the number of marks made
    struct Tree {
        lhb200::TreeDev dev; lhb200::LeafKind leaf;
        size_t copy; uint32_t item_bytes;   // the copy holding its SSZ bytes, item_bytes of them per leaf
        std::vector<uint64_t> dirty_bits; std::vector<uint32_t> dirty; uint64_t n_marks = 0;
        int list = -1;                   // index into `lists` for a resizable list
        void mark(uint64_t leaf) { dirty_bits[leaf >> 6] |= 1ull << (leaf & 63); n_marks++; }
    };
    bool incremental = false, need_full = false;
    std::vector<Tree> trees;
    uint8_t* d_levels = nullptr;
    size_t levels_bytes = 0;
    lhb200::TreeDev* d_trees = nullptr;   // trees_bytes() / dirty_bytes(), sized for `trees`
    uint32_t* d_dirty = nullptr;
    uint64_t last_root_hashes = 0;       // hash32_concat units of the last root (full or incremental)
    static constexpr uint32_t DIRTY_CAP = 1u << 16;
    // SSZ byte length of each variable-size field of the current encoding (state_layout::VAR_POS order)
    uint64_t var_len[lhb200::state_layout::N_VAR] = {};
    // Resizable lists (lhb200_state_list_edit / _set_payload_header convert a handle at its first call): each list owns
    // device storage for its items, leaf chunks and levels with headroom, and its field root comes from k_list_finish
    // instead of the tail program.
    struct List {
        int spec;                        // index into LIST_SPECS
        int tree;                        // index into `trees`
        uint64_t cap = 0;                // items the storage holds
        uint8_t* d_mem = nullptr;
        bool resized = false;            // length changed since the last root: the finishing step must run
    };
    bool converted = false;
    std::vector<List> lists;
    uint64_t units_base = 0;             // hash units of everything but the resizable lists
    std::vector<std::pair<uint32_t, uint32_t>> hdr_lits;   // payload header literals: (lit_src index, offset in header)
    int hdr_extra = -1;                  // lit_src index of extra_data
    uint32_t hdr_len_chunk = 0;          // literal chunk holding extra_data's length

    size_t trees_bytes() const { return trees.size() * sizeof(lhb200::TreeDev) + 256; }
    size_t dirty_bytes() const { return (size_t)DIRTY_CAP * 4 * trees.size(); }
    size_t coll_bytes() const { return (size_t)(shard.world + 1) * sharded.size() * 32 + 512; }
};

namespace lhb200 {

// The containers a BeaconState and a BeaconBlock share, described into a plan.  `s` = host SSZ bytes; `d` = the same
// bytes on the device, whose byte strings k_byte_items hashes in place, or null when there is no device copy (a staged
// state keeps only its big lists there): byte strings then become literal chunks, whose SSZ provenance
// lhb200_state_patch uses to find edits.  Malformed input sets `bad`.
struct SszDescriber {
    Plan& p;
    const uint8_t* s;
    const uint8_t* d;
    const ForkLayout& fl;
    bool bad = false;
    int extra_lit = -1;             // literal extra_data: its lit_src index and the literal chunk holding its length
    uint32_t extra_len_chunk = 0;

    uint64_t fail() { bad = true; return 0; }
    uint64_t u64(uint64_t off) { return p.literal_bytes(s + off, 8); }
    uint64_t h256(uint64_t off) { return p.literal_bytes(s + off, 32); }
    uint64_t addr20(uint64_t off) { return p.literal_bytes(s + off, 20); }
    uint64_t checkpoint(uint64_t off) {                                                                  // 40 B
        const uint64_t epoch = u64(off);
        return p.op_hash(epoch, h256(off + 8));
    }
    uint64_t eth1_data(uint64_t off) { return p.container({h256(off), u64(off + 32), h256(off + 40)}); }  // 72 B
    uint64_t block_header(uint64_t off) {                                                                // 112 B
        return p.container({u64(off), u64(off + 8), h256(off + 16), h256(off + 48), h256(off + 80)});
    }
    // logs_bloom: ByteVector[256]
    uint64_t bloom(uint64_t off) {
        if (d) return p.bytes_item(d + off, 256, 3, false);
        std::vector<uint64_t> chunks;
        for (int i = 0; i < 8; i++) chunks.push_back(h256(off + 32 * i));
        return p.small_tree(chunks, 3);
    }
    // extra_data: ByteList[32] at s[off, off + n)
    uint64_t extra_data(uint64_t off, uint64_t n) {
        if (d) return p.bytes_item(d + off, n, 0, true, n);
        extra_lit = (int)p.lit_src.size();
        const uint64_t chunk = p.literal_bytes(s + off, n);
        extra_len_chunk = (uint32_t)(p.lit.size() / 32);   // the next literal: mix_in_length's length
        return p.mix_in_length(chunk, n);
    }
    // The first fields of ExecutionPayload and ExecutionPayloadHeader (execution_payload.rs:54-95), extra_data checked
    // by the caller
    std::vector<uint64_t> payload_prefix(uint64_t off, Span extra) {
        return {h256(off), addr20(off + 32), h256(off + 52), h256(off + 84), bloom(off + 116), h256(off + 372),
                u64(off + 404), u64(off + 412), u64(off + 420), u64(off + 428), extra_data(off + extra.off, extra.len),
                h256(off + 440), h256(off + 472)};
    }
    // ExecutionPayloadHeader (execution_payload_header.rs:46-93): the prefix, then transactions_root, withdrawals_root,
    // blob_gas_used, excess_blob_gas, deposit_requests_root, withdrawal_requests_root up to the fork's payload field count
    uint64_t payload_header(uint64_t off, uint64_t len) {
        static constexpr struct { uint32_t off, n; } TAIL[] = {{504, 32}, {536, 32}, {568, 8}, {576, 8}, {584, 32}, {616, 32}};
        Span v[1];
        if (!read_offsets(s + off, len, fl.header_fixed, block_layout::HEADER_VAR_POS, v) || !v[0].fits(1, 32)) return fail();
        std::vector<uint64_t> f = payload_prefix(off, v[0]);
        for (int k = block_layout::PAYLOAD_PREFIX_FIELDS; k < fl.payload_fields; k++) {
            const auto& t = TAIL[k - block_layout::PAYLOAD_PREFIX_FIELDS];
            f.push_back(p.literal_bytes(s + off + t.off, t.n));
        }
        return p.container(f);
    }
};

// The resizable lists of a BeaconState, in field order (limits eth_spec.rs:389-440).  Staging checks their lengths
// against these limits and describes them with these leaf kinds; lhb200_state_list_edit resizes them.
struct ListSpec {
    uint32_t field;        // index in the state container
    int var;               // state_layout::V_*
    uint32_t item_bytes;
    uint64_t limit;        // items
    uint32_t depth;        // chunk-tree depth of the limit
    LeafKind leaf;
};
static const ListSpec LIST_SPECS[] = {
    {9, state_layout::V_VOTES, 72, 2048, 11, LEAF_ETH1_DATA},
    {11, state_layout::V_VAL, 121, 1ull << 40, 40, LEAF_VALIDATOR},
    {12, state_layout::V_BAL, 8, 1ull << 40, 38, LEAF_NONE},
    {15, state_layout::V_PP, 1, 1ull << 40, 35, LEAF_NONE},
    {16, state_layout::V_CP, 1, 1ull << 40, 35, LEAF_NONE},
    {21, state_layout::V_INACT, 8, 1ull << 40, 38, LEAF_NONE},
    {27, state_layout::V_HS, 64, 1ull << 24, 24, LEAF_CHUNK_PAIR},
    {34, state_layout::V_PBD, 16, 1ull << 27, 27, LEAF_U64_PAIR},
    {35, state_layout::V_PPW, 24, 1ull << 27, 27, LEAF_U64_TRIPLE},
    {36, state_layout::V_PC, 16, 1ull << 18, 18, LEAF_U64_PAIR},
};
constexpr int N_LIST_SPECS = sizeof(LIST_SPECS) / sizeof(LIST_SPECS[0]);
static_assert(N_LIST_SPECS <= MAX_FINISH, "one finishing thread per list");
static uint64_t list_leaves(const ListSpec& sp, uint64_t len) {
    return sp.leaf.tree == TREE_CHUNKS ? ceil_div(len * sp.item_bytes, 32) : len;
}

// Describe a whole BeaconState of any fork into `p` and the handle `st` (its copies, field and root operands, sharded
// lists, marks and header literals).  `s` = host SSZ (read for offsets and small literal fields only).  Big fields
// are placed in the arena by `place(src_off, nbytes)` which records an H2D copy.  Fields are described in order, up
// to the fork's field count, each one's plan after the previous one's (st->marks).
static int32_t describe_state(Plan& p, const uint8_t* s, uint64_t len, lhb200_state* st) {
    using namespace state_layout;
    const ShardCfg sh = st->shard;
    const ForkLayout* fl = fork_layout(sh.fork);
    if (!fl) { set_error("unknown fork id %d", sh.fork); return LHB200_EINVAL; }
    Span v[N_VAR];
    if (!read_offsets(s, len, fl->state_fixed, VAR_POS, v)) {
        set_error("BeaconState SSZ: shorter than its fixed part or inconsistent variable-part offsets");
        return LHB200_EINVAL;
    }
    bool fits = v[V_HIST].fits(32, 1u << 24);   // historical_roots: a list, but not a resizable one
    for (const ListSpec& sp : LIST_SPECS) fits = fits && v[sp.var].fits(sp.item_bytes, sp.limit);
    if (!fits) {
        set_error("BeaconState SSZ: malformed variable part");
        return LHB200_EINVAL;
    }
    const uint64_t n_hist = v[V_HIST].len / 32;
    SszDescriber c{p, s, nullptr, *fl};
    p.ssz_base = s;
    p.ssz_len = len;
    st->copies.clear();
    st->sharded.clear();
    st->marks.clear();
    st->hdr_lits.clear();
    auto place = [&](size_t src_off, size_t nbytes) -> uint8_t* {
        size_t padded = align_up(nbytes + 32, 256);
        uint8_t* d = p.alloc(padded);
        st->copies.push_back({src_off, nbytes, d, padded});
        return d;
    };
    uint64_t* f = st->field_ops;
    const uint32_t lg_world = ceil_log2(sh.world);
    // Big list with `n_chunks` leaf chunks produced from `n_items` source items of `item_bytes` at `src_off`
    // (LEAF_NONE: the bytes already are the chunks).  Unsharded: the full field root.  Sharded: this rank's subtree.
    auto big_list = [&](int field, size_t src_off, uint64_t n_items, uint32_t item_bytes, LeafKind leaf,
                        uint64_t n_chunks, uint32_t limit_depth, uint64_t mix_len) -> uint64_t {
        const uint32_t d0 = ceil_log2(std::max<uint64_t>(n_chunks, 1));
        const bool shard = sh.world > 1 && d0 >= lg_world + 6;
        const bool packed = leaf.kernel == LeafKind::NONE;
        if (!shard) {
            const uint8_t* src = place(src_off, n_items * item_bytes);
            const uint8_t* chunks = packed ? src : p.leaf_kernel(leaf, src, n_items);
            const Plan::TreeSpec warm{nullptr, 0, 0, src, leaf, st->copies.size() - 1, packed ? 32 : item_bytes};
            const uint64_t r = p.merkle_list(chunks, n_chunks, limit_depth, &warm);
            return mix_len == UINT64_MAX ? r : p.mix_in_length(r, mix_len);
        }
        const uint32_t sub = d0 - lg_world;
        const uint64_t c_lo = std::min<uint64_t>(n_chunks, (uint64_t)sh.rank << sub);
        const uint64_t c_hi = std::min<uint64_t>(n_chunks, ((uint64_t)sh.rank + 1) << sub);
        const uint64_t cnt = c_hi - c_lo;
        uint64_t op;
        if (!packed) {                 // one chunk per source item
            const uint8_t* src = place(src_off + c_lo * item_bytes, cnt * item_bytes);
            op = p.merkle_list(p.leaf_kernel(leaf, src, cnt), cnt, sub);
        } else {                       // packed bytes: chunk c covers bytes [32c, 32c+32) of the field
            const uint64_t total_bytes = n_items * item_bytes;
            const uint64_t b_lo = c_lo * 32, b_hi = std::min<uint64_t>(total_bytes, c_hi * 32);
            const uint8_t* src = place(src_off + b_lo, b_hi > b_lo ? b_hi - b_lo : 0);
            op = p.merkle_list(src, cnt, sub);
        }
        st->sharded.push_back({field, sub, limit_depth, mix_len, op});
        return Plan::zero_op(0);       // placeholder; the field root is formed in lhb200_state_combine
    };
    // a resizable list: validators and packed lists are big lists, records get one leaf-kernel root each
    auto list = [&](const ListSpec& sp) {
        const Span x = v[sp.var];
        const uint64_t n = x.len / sp.item_bytes;
        if (sp.leaf.kernel == LeafKind::VALIDATORS || sp.leaf.kernel == LeafKind::NONE)
            return big_list(sp.field, x.off, n, sp.item_bytes, sp.leaf, list_leaves(sp, n), sp.depth, n);
        return p.mix_in_length(p.merkle_list(p.leaf_kernel(sp.leaf, place(x.off, x.len), n), n, sp.depth), n);
    };
    auto plain_vector = [&](uint32_t off, uint64_t nbytes, uint32_t depth) {   // fixed vectors of chunks / packed u64
        const uint8_t* src = place(off, nbytes);
        const Plan::TreeSpec warm{nullptr, 0, 0, src, LEAF_NONE, st->copies.size() - 1, 32};
        return p.merkle_list(src, nbytes / 32, depth, &warm);
    };
    auto mark = [&] {
        PlanMark m{p.ops.size(), p.leaves.size(), st->copies.size(), p.trees.size(), p.merkle_lists.size(), {}};
        for (const auto& pass : p.passes) m.passes.push_back(pass.size());
        st->marks.push_back(std::move(m));
    };
    const ListSpec* next_list = LIST_SPECS;   // in field order
    for (int k = 0; k < fl->state_fields; k++) {   // fields 24 on: appended by later forks (beacon_state.rs:339-525)
        mark();
        if (next_list < LIST_SPECS + N_LIST_SPECS && (int)next_list->field == k) {
            f[k] = list(*next_list++);
            continue;
        }
        switch (k) {
            case 0: f[k] = c.u64(O_GENESIS_TIME); break;
            case 1: f[k] = c.h256(O_GVR); break;
            case 2: f[k] = c.u64(O_SLOT); break;
            case 3:
                f[k] = p.container({p.literal_bytes(s + O_FORK, 4), p.literal_bytes(s + O_FORK + 4, 4), c.u64(O_FORK + 8)});
                break;
            case 4: f[k] = c.block_header(O_LBH); break;
            case 5: f[k] = plain_vector(O_BLOCK_ROOTS, 8192 * 32, 13); break;
            case 6: f[k] = plain_vector(O_STATE_ROOTS, 8192 * 32, 13); break;
            case 7: f[k] = p.mix_in_length(p.merkle_list(place(v[V_HIST].off, v[V_HIST].len), n_hist, 24), n_hist); break;
            case 8: f[k] = c.eth1_data(O_ETH1_DATA); break;
            case 10: f[k] = c.u64(O_DEPOSIT_INDEX); break;
            case 13: f[k] = big_list(13, O_RANDAO, 65536, 32, LEAF_NONE, 65536, 16, UINT64_MAX); break;
            case 14: f[k] = plain_vector(O_SLASHINGS, 8192 * 8, 11); break;
            case 17: f[k] = p.literal_bytes(s + O_JUST, 1); break;
            case 18: f[k] = c.checkpoint(O_PJC); break;
            case 19: f[k] = c.checkpoint(O_CJC); break;
            case 20: f[k] = c.checkpoint(O_FC); break;
            case 22:
            case 23: {
                uint8_t* roots = p.leaf_kernel(LEAF_PUBKEY, place(k == 23 ? O_NSC : O_CSC, SYNC_COMMITTEE_BYTES), 513);
                f[k] = p.container({p.merkle_list(roots, 512, 9), reinterpret_cast<uint64_t>(roots + 512 * 32)});
                break;
            }
            case 24: {   // its literals move when an earlier list changes length, and are rewritten by a new header
                const size_t l0 = p.lit_src.size();
                f[k] = c.payload_header(v[V_LEPH].off, v[V_LEPH].len);
                for (size_t i = l0; i < p.lit_src.size(); i++)
                    st->hdr_lits.push_back({(uint32_t)i, (uint32_t)(p.lit_src[i].src_off - v[V_LEPH].off)});
                break;
            }
            case 25: f[k] = c.u64(O_NWI); break;
            case 26: f[k] = c.u64(O_NWVI); break;
            default: f[k] = c.u64(O_ELECTRA_U64 + 8 * (k - 28)); break;   // 28 .. 33
        }
    }
    mark();
    if (c.bad) { set_error("BeaconState SSZ: malformed execution payload header"); return LHB200_EINVAL; }
    st->hdr_extra = c.extra_lit;
    st->hdr_len_chunk = c.extra_len_chunk;
    for (int k = fl->state_fields; k < MAX_FIELDS; k++) f[k] = Plan::zero_op(0);   // absent in this fork (not part of its container)
    st->root_op = p.container(std::vector<uint64_t>(f, f + fl->state_fields));
    return LHB200_OK;
}

__global__ void k_gather_nodes(const HashOp* __restrict__ srcs, int n, uint8_t* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
    load_operand(srcs[i].a, w);
    store_chunk(out + 32 * i, w);
}

// Operand table of k_gather_nodes, staged through the pinned `h` (n * sizeof(HashOp) bytes).
static int32_t stage_operands(const std::vector<uint64_t>& operands, HashOp* d_tab, uint8_t* h, cudaStream_t s) {
    HashOp* tab = reinterpret_cast<HashOp*>(h);
    for (size_t i = 0; i < operands.size(); i++) tab[i] = {0, operands[i], 0};
    LHB_CUDA(cudaMemcpyAsync(d_tab, tab, operands.size() * sizeof(HashOp), cudaMemcpyHostToDevice, s));
    return LHB200_OK;
}
// The n operands a staged table lists -> n contiguous chunks at `out`.
static int32_t gather_operands(const HashOp* d_tab, uint32_t n, uint8_t* out, cudaStream_t s) {
    k_gather_nodes<<<(unsigned)ceil_div(n, 64), 64, 0, s>>>(d_tab, (int)n, out);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    return LHB200_OK;
}

// The resident parts [a, b) of SSZ bytes [lo, hi) of a staged state: on_copy(copy index, a, b) for staged copies,
// on_lit(literal source, a, b) for literal chunks, each returning whether to go on; returns whether there were any.
// Each kind is found by binary search over offset-sorted indices: O(log fields) per edit, so a slot's worth of
// mutations (tens of thousands of 8-byte edits) costs the host well under a millisecond.  `hint`, the copy of the
// previous edit, is tried first.
template <class C, class L>
static bool visit_resident(const lhb200_state* st, uint64_t lo, uint64_t hi, size_t& hint, C&& on_copy, L&& on_lit) {
    bool any = false;
    const std::vector<uint32_t>& co = st->copy_order;
    auto before = [&](uint32_t ci) { return st->copies[ci].src_off + st->copies[ci].nbytes <= lo; };
    size_t k = hint < co.size() && st->copies[co[hint]].src_off <= lo && !before(co[hint])
                   ? hint : std::partition_point(co.begin(), co.end(), before) - co.begin();
    for (hint = k; k < co.size() && st->copies[co[k]].src_off < hi; k++) {
        const StageCopy& cp = st->copies[co[k]];
        const uint64_t a = std::max<uint64_t>(lo, cp.src_off), b = std::min<uint64_t>(hi, cp.src_off + cp.nbytes);
        if (a >= b) continue;
        any = true;
        if (!on_copy(co[k], a, b)) return true;
    }
    const std::vector<Plan::LitSrc>& ls = st->plan.lit_src;
    const std::vector<uint32_t>& lo_order = st->lit_order;
    size_t m = std::partition_point(lo_order.begin(), lo_order.end(),
                                    [&](uint32_t li) { return ls[li].src_off + ls[li].n <= lo; }) - lo_order.begin();
    for (; m < lo_order.size() && ls[lo_order[m]].src_off < hi; m++) {
        const Plan::LitSrc& l = ls[lo_order[m]];
        const uint64_t a = std::max<uint64_t>(lo, l.src_off), b = std::min<uint64_t>(hi, l.src_off + l.n);
        if (a >= b) continue;
        any = true;
        if (!on_lit(l, a, b)) return true;
    }
    return any;
}
// Offset order of a handle's copies and literals, and copy_tree: rebuilt whenever offsets move or trees change
// (staging, lhb200_state_enable_incremental, list and header edits).  An empty range sorts before a range that starts
// at the same offset (an empty list and the next field), so that the ends ascend too, as visit_resident's binary
// search needs.
static void index_resident(lhb200_state* st) {
    const std::vector<StageCopy>& cp = st->copies;
    st->copy_order.resize(cp.size());
    for (size_t k = 0; k < cp.size(); k++) st->copy_order[k] = (uint32_t)k;
    std::sort(st->copy_order.begin(), st->copy_order.end(), [&](uint32_t a, uint32_t b) {
        return cp[a].src_off != cp[b].src_off ? cp[a].src_off < cp[b].src_off : cp[a].nbytes < cp[b].nbytes;
    });
    const std::vector<Plan::LitSrc>& ls = st->plan.lit_src;
    st->lit_order.resize(ls.size());
    for (size_t k = 0; k < ls.size(); k++) st->lit_order[k] = (uint32_t)k;
    std::sort(st->lit_order.begin(), st->lit_order.end(), [&](uint32_t a, uint32_t b) {
        return ls[a].src_off != ls[b].src_off ? ls[a].src_off < ls[b].src_off : ls[a].n < ls[b].n;
    });
    st->copy_tree.assign(st->copies.size(), -1);
    for (size_t t = 0; t < st->trees.size(); t++) st->copy_tree[st->trees[t].copy] = (int32_t)t;
}

// ---------------------------------------------------------------------------------------------------------
// Merkle proofs by generalized index (consensus-specs ssz/merkle-proofs.md; BeaconState::compute_merkle_proof,
// beacon_state.rs:2483-2557; BeaconBlockBody::kzg_commitment_merkle_proof, beacon_block_body.rs:178-227).  A gindex g
// names the node at depth floor(log2 g) below a root; its branch lists the siblings along the path, bottom-up.  The
// host walks g's bits from the root through what the describer emitted:
//   - an op output: bit 0 goes to operand a, bit 1 to operand b, the other operand is the sibling;
//   - a zero operand: the rest of the path lies in a zero subtree, whose siblings are zero hashes;
//   - the top of a resident tree (an incremental handle's big lists) or of a merkle_list folded by reduce passes, whose
//     levels are rebuilt into per-call scratch: the rest of the path is a leaf index into the tree's levels;
//   - the field root of a converted resizable list, which k_list_finish writes with no op behind it: its length chunk
//     and its ladder above the current top are synthesised, the left spine node a right turn above the top needs is
//     hashed by k_proof_branches from the top node;
//   - anything else is a leaf (a literal, a validator, record or byte-item root): a further bit is refused.
// The siblings above the point where a path enters a tree are listed once per such entry node (of one root), and
// later proofs that enter the same node below the same root (100 000 validator proofs) reuse them: per proof the host
// then only computes a leaf index.
constexpr uint64_t PROOF_IMM = 1ull << 62;   // ProofSrc::op until upload: index of an immediate chunk (a list length)

struct ProofResolver {
    const Plan& pl;
    std::vector<std::pair<uint64_t, const TreeDev*>> resident;    // top node address -> tree with resident levels
    std::vector<std::pair<uint64_t, const TreeDev*>> converted;   // field root address -> converted resizable list
    // output: proofs, first[k] = siblings of proofs [0, k), sibling sources above the trees, immediate chunks, and the
    // trees the proofs enter (resident levels, or a merkle_list whose levels this call rebuilds)
    std::vector<ProofDesc> desc;
    std::vector<uint64_t> first{0};
    std::vector<ProofSrc> srcs;
    std::vector<std::array<uint8_t, 32>> imm;
    struct TreeUse { const TreeDev* dev; const Plan::ListRec* rec; };
    std::vector<TreeUse> trees;

    static constexpr uint32_t NONE = ~0u;
    std::vector<uint32_t> pool_op, forced_op;   // node-pool slot / forced destination -> the op writing it
    struct Entry { uint32_t tree, top, src; };  // a tree entry node: its tree and the siblings above it
    // by (the root the walk started from, the entry node's gindex below it): the blocks of a batch share gindices but
    // not trees or siblings
    struct MemoKey {
        uint64_t root, g;
        bool operator==(const MemoKey& o) const { return root == o.root && g == o.g; }
    };
    struct MemoHash {
        size_t operator()(const MemoKey& k) const { return std::hash<uint64_t>()(k.g ^ (k.root * 0x9e3779b97f4a7c15ull)); }
    };
    std::unordered_map<MemoKey, Entry, MemoHash> memo;
    std::vector<uint32_t> memo_depths;

    explicit ProofResolver(const Plan& p) : pl(p) {
        pool_op.assign(p.node_used, NONE);
        forced_op.assign(p.forced_wave.size(), NONE);
        for (size_t i = 0; i < p.ops.size(); i++) {
            const uint64_t dst = p.ops[i].dst, s = (dst - reinterpret_cast<uint64_t>(p.arena) - p.node_off) / 32;
            if (s < pool_op.size()) pool_op[s] = (uint32_t)i;
            else if ((dst - p.forced_base) / 32 < forced_op.size()) forced_op[(dst - p.forced_base) / 32] = (uint32_t)i;
        }
    }
    // the resident trees and converted lists of a state handle
    void add_state(const lhb200_state* st) {
        for (const lhb200_state::Tree& t : st->trees) {
            if (t.list >= 0) converted.push_back({reinterpret_cast<uint64_t>(t.dev.field_dst), &t.dev});
            else resident.push_back({reinterpret_cast<uint64_t>(t.dev.top_dst), &t.dev});
        }
    }
    uint32_t producer(uint64_t a) const {
        const uint64_t off = a - reinterpret_cast<uint64_t>(pl.arena) - pl.node_off;   // outside the pool: huge
        if (off % 32 == 0 && off / 32 < pool_op.size()) return pool_op[off / 32];
        const uint64_t f = a - pl.forced_base;
        if (f % 32 == 0 && f / 32 < forced_op.size()) return forced_op[f / 32];
        return NONE;
    }
    static const TreeDev* find(const std::vector<std::pair<uint64_t, const TreeDev*>>& v, uint64_t a) {
        for (const auto& e : v)
            if (e.first == a) return e.second;
        return nullptr;
    }
    uint32_t tree_id(const TreeDev* dev, const Plan::ListRec* rec) {
        for (size_t k = 0; k < trees.size(); k++)
            if (trees[k].dev == dev && trees[k].rec == rec) return (uint32_t)k;
        trees.push_back({dev, rec});
        return (uint32_t)trees.size() - 1;
    }
    static ProofSrc zero(uint32_t l) { return {OP_ZERO_FLAG | l, 0, 0}; }
    // the left spine node of a non-empty converted list at level l >= top: its top node laddered with zero hashes
    static ProofSrc spine(const TreeDev& t, uint32_t l) { return {reinterpret_cast<uint64_t>(t.lvl[t.top]), t.top, l}; }

    void push(uint64_t node, uint32_t tree, uint32_t level, uint32_t n_tree, uint32_t src, uint32_t depth) {
        desc.push_back({node, tree, level, n_tree, src});
        first.push_back(first.back() + depth);
    }
    static int32_t refuse(uint64_t g, const char* why) {
        set_error("merkle proof: gindex %llu: %s", (unsigned long long)g, why);
        return LHB200_EINVAL;
    }

    // Resolve gindex g below the node `root` into one more proof.
    int32_t resolve(uint64_t root, uint64_t g) {
        if (g == 0) return refuse(g, "0 is not a generalized index");
        const uint32_t D = 63 - (uint32_t)__builtin_clzll(g);
        for (uint32_t d : memo_depths) {
            if (d > D) continue;
            const auto it = memo.find({root, g >> (D - d)});
            if (it == memo.end()) continue;
            const Entry& e = it->second;
            if (D - d > e.top) return refuse(g, "below a leaf");
            push(g & ((1ull << (D - d)) - 1), e.tree, e.top - (D - d), D - d, e.src, D);
            return LHB200_OK;
        }
        std::vector<ProofSrc> up;   // siblings so far, top-down
        uint64_t cur = root;
        const TreeDev* list = nullptr;   // inside a converted list: at its field root (level limit_depth + 1) or on
        uint32_t level = 0;              // its left spine at `level`
        bool leaf = false;
        auto enter = [&](uint32_t tree, uint32_t top, uint32_t r) {   // the remaining r bits index the tree's levels
            if (r > top) return refuse(g, "below a leaf");
            const uint32_t src = (uint32_t)srcs.size();
            srcs.insert(srcs.end(), up.rbegin(), up.rend());
            memo[{root, g >> r}] = {tree, top, src};
            if (std::find(memo_depths.begin(), memo_depths.end(), D - r) == memo_depths.end()) memo_depths.push_back(D - r);
            push(g & ((1ull << r) - 1), tree, top - r, r, src, D);
            return LHB200_OK;
        };
        for (int k = (int)D - 1; k >= 0; k--) {
            const uint32_t bit = (g >> k) & 1, r = (uint32_t)k + 1;   // r levels left below the current node
            if (leaf) return refuse(g, "below a leaf");
            if (!list && !(cur & OP_ZERO_FLAG)) {
                const uint32_t i = producer(cur);
                if (i != NONE) {
                    const HashOp& op = pl.ops[i];
                    up.push_back({bit ? op.a : op.b, 0, 0});
                    cur = bit ? op.b : op.a;
                    continue;
                }
                if (const TreeDev* t = find(resident, cur)) return enter(tree_id(t, nullptr), t->top, r);
                if ((list = find(converted, cur))) {
                    level = list->limit_depth + 1;
                } else {
                    for (const Plan::ListRec& lr : pl.merkle_lists)
                        if (lr.top_addr == cur) return enter(tree_id(nullptr, &lr), ceil_log2(lr.n), r);
                    return refuse(g, "below a leaf");
                }
            }
            if (list) {
                const TreeDev& t = *list;
                if (level == t.top && t.n_leaves) return enter(tree_id(list, nullptr), t.top, r);
                if (level > t.limit_depth) {   // field root = H(data root, length chunk)
                    if (bit) {
                        up.push_back(t.n_leaves ? spine(t, t.limit_depth) : zero(t.limit_depth));
                        leaf = true;
                        continue;
                    }
                    std::array<uint8_t, 32> len{};
                    for (int b = 0; b < 8; b++) len[b] = (uint8_t)(t.length >> (8 * b));
                    up.push_back({PROOF_IMM | imm.size(), 0, 0});
                    imm.push_back(len);
                    if (t.n_leaves) { level = t.limit_depth; } else { list = nullptr; cur = OP_ZERO_FLAG | t.limit_depth; }
                    continue;
                }
                // on the left spine above the top: a left turn stays on it, a right turn enters a zero subtree
                up.push_back(bit ? spine(t, level - 1) : zero(level - 1));
                if (bit) { list = nullptr; cur = OP_ZERO_FLAG | (level - 1); }
                level--;
                continue;
            }
            const uint32_t z = (uint32_t)(cur & 0xff);   // a zero subtree of height z
            if (r > z) return refuse(g, "below a leaf");
            for (uint32_t l = z; l > z - r; l--) up.push_back(zero(l - 1));
            break;
        }
        const uint32_t src = (uint32_t)srcs.size();
        srcs.insert(srcs.end(), up.rbegin(), up.rend());
        push(0, 0, 0, 0, src, D);
        return LHB200_OK;
    }

    // Bytes of the tables (pinned staging and device alike), then of the rebuilt levels and of the branches.
    size_t table_bytes() const {
        return align_up(desc.size() * sizeof(ProofDesc), 256) + align_up(first.size() * 8, 256) +
               align_up(srcs.size() * sizeof(ProofSrc), 256) + align_up(imm.size() * 32, 256) +
               align_up(trees.size() * sizeof(ProofTree), 256);
    }
    size_t levels_bytes() const {
        size_t b = 0;
        for (const TreeUse& u : trees)
            if (u.rec)
                for (uint64_t n = u.rec->n, l = 1; l < ceil_log2(u.rec->n); l++) b += align_up((n = ceil_div(n, 2)) * 32, 256);
        return b;
    }
    size_t device_bytes() const { return table_bytes() + levels_bytes() + align_up(first.back() * 32, 256) + 256; }

    // Device state of one call: the tables at `d` (device_bytes()), staged through the pinned `h` (table_bytes()).
    ProofDesc* d_desc = nullptr;
    uint64_t* d_first = nullptr;
    ProofSrc* d_srcs = nullptr;
    ProofTree* d_trees = nullptr;
    uint8_t* d_branches = nullptr;
    std::vector<ProofTree> tabs;
    int32_t upload(uint8_t* h, uint8_t* d, cudaStream_t s) {
        size_t o = 0;
        auto put = [&](const void* src, size_t bytes) {
            uint8_t* p = d + o;
            if (bytes) memcpy(h + o, src, bytes);
            o += align_up(bytes, 256);
            return p;
        };
        d_desc = reinterpret_cast<ProofDesc*>(put(desc.data(), desc.size() * sizeof(ProofDesc)));
        d_first = reinterpret_cast<uint64_t*>(put(first.data(), first.size() * 8));
        const size_t o_srcs = o;
        d_srcs = reinterpret_cast<ProofSrc*>(put(srcs.data(), srcs.size() * sizeof(ProofSrc)));
        uint8_t* d_imm = put(imm.data(), imm.size() * 32);
        for (size_t i = 0; i < srcs.size(); i++) {   // immediates: now that they have an address
            ProofSrc& x = reinterpret_cast<ProofSrc*>(h + o_srcs)[i];
            if (!(x.op & OP_ZERO_FLAG) && (x.op & PROOF_IMM)) x.op = reinterpret_cast<uint64_t>(d_imm + 32 * (x.op & ~PROOF_IMM));
        }
        uint8_t* lv = d + table_bytes();   // rebuilt levels, laid out as levels_bytes() counts them
        tabs.assign(trees.size(), ProofTree{});
        for (size_t k = 0; k < trees.size(); k++) {
            ProofTree& pt = tabs[k];
            if (trees[k].dev) {
                for (int l = 0; l < 41; l++) pt.lvl[l] = trees[k].dev->lvl[l];
                pt.n_leaves = trees[k].dev->n_leaves;
                continue;
            }
            const Plan::ListRec& lr = *trees[k].rec;
            pt.lvl[0] = lr.chunks;
            pt.n_leaves = lr.n;
            uint64_t n = lr.n;
            for (uint32_t l = 1; l < ceil_log2(lr.n); l++) {
                pt.lvl[l] = lv;
                lv += align_up((n = ceil_div(n, 2)) * 32, 256);
            }
        }
        d_trees = reinterpret_cast<ProofTree*>(put(tabs.data(), tabs.size() * sizeof(ProofTree)));
        d_branches = lv;
        LHB_CUDA(cudaMemcpyAsync(d, h, o, cudaMemcpyHostToDevice, s));
        return LHB200_OK;
    }
    // After the root: rebuild the levels of the merkle_lists the proofs enter (one k_tree_level launch per level), then
    // gather every sibling (one k_proof_branches launch).  e0 / e1 (optional) are recorded around the gather.
    int32_t enqueue(cudaStream_t s, cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr) const {
        for (size_t k = 0; k < trees.size(); k++) {
            if (!trees[k].rec) continue;
            uint64_t n = trees[k].rec->n;
            for (uint32_t l = 0; l + 2 <= ceil_log2(trees[k].rec->n); l++) {
                k_tree_level<<<(unsigned)ceil_div(ceil_div(n, 2), 256), 256, 0, s>>>(tabs[k].lvl[l], n,
                                                                                    const_cast<uint8_t*>(tabs[k].lvl[l + 1]), l);
                count_launch();
                n = ceil_div(n, 2);
            }
        }
        const uint64_t total = first.back();
        if (e0) cudaEventRecord(e0, s);
        if (total) {
            k_proof_branches<<<(unsigned)ceil_div(total, 256), 256, 0, s>>>(d_desc, d_first, (uint32_t)desc.size(), d_trees,
                                                                           d_srcs, d_branches);
            count_launch();
        }
        if (e1) cudaEventRecord(e1, s);
        LHB_CUDA(cudaGetLastError());
        return LHB200_OK;
    }
};

}  // namespace lhb200

using namespace lhb200;

extern "C" {

int32_t lhb200_hash_pairs(const uint8_t* in, uint8_t* out, uint64_t n) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!in || !out) { set_error("null buffer"); return LHB200_EINVAL; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(n * 96 + 512));
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(n * 96));
    if (!d || !h) return LHB200_ENOMEM;
    memcpy(h, in, n * 64);
    LHB_CUDA(cudaMemcpyAsync(d, h, n * 64, cudaMemcpyHostToDevice, c.stream));
    uint8_t* d_out = d + align_up(n * 64, 256);
    k_hash_pairs<<<(unsigned)ceil_div(n, 256), 256, 0, c.stream>>>(d, d_out, n);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(h + n * 64, d_out, n * 32, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out, h + n * 64, n * 32);
    return LHB200_OK;
}

int32_t lhb200_dev_hash_pairs(const void* d_in, void* d_out, uint64_t n, void* stream) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!d_in || !d_out || (reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15)) {
        set_error("device buffers must be non-null and 16-byte aligned");
        return LHB200_EINVAL;
    }
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    k_hash_pairs<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(static_cast<const uint8_t*>(d_in),
                                                           static_cast<uint8_t*>(d_out), n);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    return LHB200_OK;
}

int32_t lhb200_merkleize(const uint8_t* chunks, uint64_t n_chunks, uint32_t depth, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    if (!out || (n_chunks && !chunks) || depth > 64 || (depth < 64 && n_chunks > (1ull << depth))) {
        set_error("merkleize: bad arguments (n_chunks must be <= 2^depth, depth <= 64)");
        return LHB200_EINVAL;
    }
    return run_simple(chunks, n_chunks * 32, out,
                      [&](Plan& p, uint8_t* d_in) { return p.merkle_list(d_in, n_chunks, depth); });
}

int32_t lhb200_dev_merkleize(const void* d_chunks, uint64_t n_chunks, uint32_t depth, void* d_out32, void* stream) {
    LHB_REQUIRE_READY();
    if (!d_out32 || (n_chunks && !d_chunks) || (reinterpret_cast<uintptr_t>(d_chunks) & 15) ||
        (reinterpret_cast<uintptr_t>(d_out32) & 15) || depth > 64 || (depth < 64 && n_chunks > (1ull << depth))) {
        set_error("dev_merkleize: bad arguments");
        return LHB200_EINVAL;
    }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c.stream;
    uint64_t root = 0;
    Plan pl;
    int32_t rc = build_sized(pl, 256, 256, [&](Plan& p) {
        root = p.merkle_list(static_cast<const uint8_t*>(d_chunks), n_chunks, depth);
        return LHB200_OK;
    }, scratch_arena);
    if (rc) return rc;
    const size_t hr = align_up(plan_stage_bytes(pl), 256);
    uint8_t* hst = static_cast<uint8_t*>(pinned_scratch(hr + 32));
    if (!hst) return LHB200_ENOMEM;
    rc = plan_upload(pl, s, hst);
    if (rc) return rc;
    rc = plan_enqueue(pl, s);
    if (rc) return rc;
    rc = read_root(root, d_out32, cudaMemcpyDeviceToDevice, hst + hr, s);
    if (rc) return rc;
    // the scratch arena and pinned staging are reused by the next call: finish before returning
    LHB_CUDA(cudaStreamSynchronize(s));
    return LHB200_OK;
}

int32_t lhb200_mix_in_length(const uint8_t root[32], uint64_t len, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    if (!root || !out) return LHB200_EINVAL;
    return run_simple(root, 32, out, [&](Plan& p, uint8_t* d_in) {
        return p.mix_in_length(reinterpret_cast<uint64_t>(d_in), len);
    });
}

int32_t lhb200_zero_hash(uint32_t depth, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    if (depth > 64 || !out) return LHB200_EINVAL;
    memcpy(out, ctx().zero_hashes[depth], 32);
    return LHB200_OK;
}

int32_t lhb200_validators_root(const uint8_t* ssz, uint64_t n, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    if (!out || (n && !ssz) || n > (1ull << 40)) return LHB200_EINVAL;
    return run_simple(ssz, n * 121, out, [&](Plan& p, uint8_t* d_in) {
        return p.mix_in_length(p.merkle_list(p.leaf_kernel(LEAF_VALIDATOR, d_in, n), n, 40), n);
    });
}

int32_t lhb200_validator_roots(const uint8_t* ssz, uint64_t n, uint8_t* out_roots) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!ssz || !out_roots) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    size_t in_pad = align_up(n * 121, 256);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(in_pad + n * 32 + 256));
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(n * 121 + n * 32));
    if (!d || !h) return LHB200_ENOMEM;
    memcpy(h, ssz, n * 121);
    LHB_CUDA(cudaMemcpyAsync(d, h, n * 121, cudaMemcpyHostToDevice, c.stream));
    k_validator_roots<<<(unsigned)ceil_div(n, VAL_PER_CTA), VAL_PER_CTA, 0, c.stream>>>(d, n, d + in_pad);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(h + n * 121, d + in_pad, n * 32, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out_roots, h + n * 121, n * 32);
    return LHB200_OK;
}

static int32_t stage_state(const uint8_t* ssz, uint64_t len, ShardCfg sh, lhb200_state** out) {
    LHB_REQUIRE_READY();
    if (!ssz || !out) return LHB200_EINVAL;
    if (sh.world == 0 || (sh.world & (sh.world - 1)) || sh.rank >= sh.world) {
        set_error("state shard: world must be a power of two and rank < world");
        return LHB200_EINVAL;
    }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    // a failure releases the handle, which keeps the arena it took as the spare for the next stage call
    std::unique_ptr<lhb200_state, int32_t (*)(lhb200_state*)> st(new lhb200_state(), lhb200_state_release);
    st->shard = sh;
    constexpr size_t n_result = 1 + MAX_FIELDS;
    int32_t rc = build_sized(st->plan, 16384, n_result * 32 + n_result * sizeof(HashOp) + 1024, [&](Plan& p) {
        return describe_state(p, ssz, len, st.get());
    }, [&](size_t need, uint8_t** arena, size_t* bytes) {
        if (g_spare_arena && g_spare_bytes >= need) {   // recycled from the last released handle (no cudaMalloc)
            st->arena = g_spare_arena;
            st->arena_bytes = g_spare_bytes;
            g_spare_arena = nullptr;
            g_spare_bytes = 0;
        } else {
            uint8_t* a = nullptr;
            LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&a), need + (need >> 3)));
            st->arena = a;
            st->arena_bytes = need + (need >> 3);
        }
        *arena = st->arena;
        *bytes = st->arena_bytes;
        return LHB200_OK;
    });
    if (rc) return rc;
    {   // the describer has checked the offsets
        Span v[state_layout::N_VAR];
        read_offsets(ssz, len, fork_layout(sh.fork)->state_fixed, state_layout::VAR_POS, v);
        for (int k = 0; k < state_layout::N_VAR; k++) st->var_len[k] = v[k].len;
    }
    st->plan.ssz_base = nullptr;  // the caller's buffer is not retained
    // allocated before the program blobs, so that plan_upload's arena check covers them too
    std::vector<uint64_t> gather(1, st->root_op);   // root + field roots -> contiguous result block
    gather.insert(gather.end(), st->field_ops, st->field_ops + MAX_FIELDS);
    for (const ShardedList& L : st->sharded) gather.push_back(L.local_op);
    st->d_gather = reinterpret_cast<HashOp*>(st->plan.alloc(gather.size() * sizeof(HashOp)));
    st->d_result = st->plan.alloc(n_result * 32);
    const HostInput in(ssz, len);
    const size_t hp = in.bounce_bytes(), hg = hp + align_up(plan_stage_bytes(st->plan), 256);
    uint8_t* hst = static_cast<uint8_t*>(pinned_scratch(hg + gather.size() * sizeof(HashOp)));
    if (!hst) return LHB200_ENOMEM;
    // H2D: per-field copies into the aligned layout
    const uint8_t* src = in.source(hst);
    for (const StageCopy& cp : st->copies) {
        size_t z0 = cp.nbytes / 256 * 256;
        LHB_CUDA(cudaMemsetAsync(cp.dst + z0, 0, cp.pad_to - z0, c.stream));
        if (cp.nbytes)
            LHB_CUDA(cudaMemcpyAsync(cp.dst, src + cp.src_off, cp.nbytes, cudaMemcpyHostToDevice, c.stream));
    }
    rc = plan_upload(st->plan, c.stream, hst + hp);
    if (rc) return rc;
    rc = stage_operands(gather, st->d_gather, hst + hg, c.stream);
    if (rc) return rc;
    index_resident(st.get());
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    *out = st.release();
    return LHB200_OK;
}

int32_t lhb200_state_stage_deneb(const uint8_t* ssz, uint64_t len, lhb200_state** out) {
    return stage_state(ssz, len, ShardCfg(), out);
}
// Same for any post-Altair fork (LHB200_FORK_*): the describer is table-driven, the kernels are shared.
int32_t lhb200_state_stage(const uint8_t* ssz, uint64_t len, int32_t fork, lhb200_state** out) {
    ShardCfg sh;
    sh.fork = fork;
    return stage_state(ssz, len, sh, out);
}

int32_t lhb200_state_stage_deneb_shard(const uint8_t* ssz, uint64_t len, uint32_t rank, uint32_t world,
                                       lhb200_state** out) {
    ShardCfg sh;
    sh.rank = rank;
    sh.world = world;
    return stage_state(ssz, len, sh, out);
}

// Run this rank's part and return the subtree roots of the sharded lists (n_lists x 32 bytes, fixed list order).
int32_t lhb200_state_shard_roots(lhb200_state* st, uint8_t* out, uint32_t* n_lists) {
    LHB_REQUIRE_READY();
    if (!st || !out || !n_lists) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    int32_t rc = lhb200_state_root_enqueue(st, c.stream, nullptr);
    if (rc) return rc;
    const uint32_t n = (uint32_t)st->sharded.size();
    *n_lists = n;
    if (n == 0) { LHB_CUDA(cudaStreamSynchronize(c.stream)); return LHB200_OK; }
    uint8_t* h_res = static_cast<uint8_t*>(pinned_scratch(n * 32));
    uint8_t* d_res = static_cast<uint8_t*>(dev_scratch(n * 32));
    if (!h_res || !d_res) return LHB200_ENOMEM;
    rc = gather_operands(st->d_gather + 1 + MAX_FIELDS, n, d_res, c.stream);
    if (rc) return rc;
    LHB_CUDA(cudaMemcpyAsync(h_res, d_res, n * 32, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out, h_res, n * 32);
    return LHB200_OK;
}

// Fold the all-gathered subtree roots (rank-major: gathered[(g * n_lists + l) * 32]) into the state root.
// Must be called after lhb200_state_shard_roots on the same handle (the unsharded field roots live in its arena).
static int32_t state_combine_impl(lhb200_state* st, const uint8_t* gathered, uint8_t out[32], bool on_device) {
    if (!st || !gathered || !out) return LHB200_EINVAL;
    const uint32_t n = (uint32_t)st->sharded.size(), world = st->shard.world;
    uint32_t lg = 0;
    while ((1u << lg) < world) lg++;
    return run_simple(gathered, (size_t)world * n * 32, out, [&](Plan& p, uint8_t* d_in) {
        std::vector<uint64_t> f(st->field_ops, st->field_ops + 28);   // (sharded handles are Deneb: 28 fields)
        for (uint32_t l = 0; l < n; l++) {
            const ShardedList& L = st->sharded[l];
            std::vector<uint64_t> nodes;
            for (uint32_t gidx = 0; gidx < world; gidx++)
                nodes.push_back(reinterpret_cast<uint64_t>(d_in + ((size_t)gidx * n + l) * 32));
            uint64_t r = p.small_tree(nodes, lg);
            for (uint32_t d = L.s + lg; d < L.limit_depth; d++) r = p.op_hash(r, Plan::zero_op(d));
            if (L.mix_len != UINT64_MAX) r = p.mix_in_length(r, L.mix_len);
            f[L.field] = r;
        }
        return p.container(f);
    }, on_device);
}
int32_t lhb200_state_combine(lhb200_state* st, const uint8_t* gathered, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    return state_combine_impl(st, gathered, out, false);
}

// One BeaconState root over the ranks of the library's communicator (lhb200_comm_init), on a handle staged with
// lhb200_state_stage_deneb_shard(rank, world): the shard's subtree roots stay on the device, one ncclAllGather of
// n_lists x 32 B per rank, then every rank folds the top (log2(world) levels, zero ladders, length mix-ins, container)
// — all on the library's stream; the only host transfer is the 32-byte root (SURVEY.md §8e "Tree hash").
int32_t lhb200_state_root_sharded(lhb200_state* st, uint8_t out[32]) {
    LHB_REQUIRE_READY();
    if (!st || !out) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const uint32_t n = (uint32_t)st->sharded.size(), world = st->shard.world;
    if ((int)world != comm_world() && world != 1) { set_error("state sharded %u ways but the communicator has %d ranks", world, comm_world()); return LHB200_EINVAL; }
    int32_t rc = lhb200_state_root_enqueue(st, c.stream, nullptr);
    if (rc) return rc;
    if (n == 0) { set_error("handle is not sharded"); return LHB200_EINVAL; }
    if (!st->d_coll) {   // owned by the handle: dev_scratch is reused by the combine
        LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_coll), st->coll_bytes()));
    }
    uint8_t* d_mine = st->d_coll;
    uint8_t* d_all = d_mine + align_up(n * 32, 256);
    rc = gather_operands(st->d_gather + 1 + MAX_FIELDS, n, d_mine, c.stream);
    if (rc) return rc;
    rc = comm_allgather_bytes(d_mine, d_all, (size_t)n * 32, c.stream);
    if (rc) return rc;
    return state_combine_impl(st, d_all, out, true);
}

// Apply same-length mutations to a staged state (the resident analogue of BeaconState::apply_pending_mutations,
// consensus/types/src/beacon_state.rs:2459-2481): `data` replaces SSZ bytes [ssz_offset, ssz_offset + len) of the
// encoding the handle was staged from.  Big-field bytes are patched in place in HBM, small-field bytes re-pack their
// literal chunks.  List lengths / variable-part offsets must not change (re-stage for that).  The next
// lhb200_state_root re-hashes the whole state (cheaper than tracking dirty paths unless incremental mode is enabled).
// n same-length mutations in one call: offsets[i], lens[i], bytes concatenated in `data`.  Ranges must not overlap.
// One H2D copy of the blob + one scatter kernel; dirty leaves are recorded for the warm path.
int32_t lhb200_state_patch_batch(lhb200_state* st, const uint64_t* offsets, const uint32_t* lens, const uint8_t* data,
                                 uint32_t n) {
    LHB_REQUIRE_READY();
    if (!st || (n && (!offsets || !lens || !data))) return LHB200_EINVAL;
    if (n == 0) return LHB200_OK;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) total += lens[i];
    std::vector<ScatterOp> ops;
    ops.reserve(n);
    Plan& pl = st->plan;
    uint32_t lit_lo = ~0u, lit_hi = 0;
    // pass 1: every edit must hit resident bytes — validated BEFORE anything is modified, so a rejected batch leaves the
    // handle (host literals, dirty lists, device copy) exactly as it was
    auto stop = [](auto&&...) { return false; };
    size_t hint = ~(size_t)0;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t lo = offsets[i], hi = lo + lens[i];
        if (lens[i] && !visit_resident(st, lo, hi, hint, stop, stop)) {
            set_error("state_patch: range [%llu, %llu) is not resident on this handle (offset table or another rank's shard)",
                      (unsigned long long)lo, (unsigned long long)hi);
            return LHB200_EINVAL;
        }
    }
    uint64_t blob_off = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t lo = offsets[i], hi = lo + lens[i];
        const uint8_t* src = data + blob_off;
        visit_resident(st, lo, hi, hint, [&](uint32_t ci, uint64_t a, uint64_t b) {
            const StageCopy& cp = st->copies[ci];
            ops.push_back({cp.dst + (a - cp.src_off), (uint32_t)(b - a), (uint32_t)(blob_off + (a - lo))});
            if (!st->incremental || st->need_full) return true;   // warm path: which leaves of which tree does this touch?
            const int32_t ti = st->copy_tree[ci];
            if (ti < 0) { st->need_full = true; return true; }     // a list without a resident tree (votes, summaries, ...)
            lhb200_state::Tree& t = st->trees[ti];
            const uint64_t i0 = (a - cp.src_off) / t.item_bytes, i1 = (b - 1 - cp.src_off) / t.item_bytes;
            if (t.n_marks + (i1 - i0 + 1) > 4ull * lhb200_state::DIRTY_CAP) { st->need_full = true; return true; }
            for (uint64_t q = i0; q <= i1; q++) t.mark(q);
            return true;
        }, [&](const Plan::LitSrc& ls, uint64_t a, uint64_t b) {   // small fixed fields live in host-packed literal chunks
            memcpy(&pl.lit[(size_t)ls.lit_index * 32] + (a - ls.src_off), src + (a - lo), b - a);
            lit_lo = std::min(lit_lo, ls.lit_index);
            lit_hi = std::max(lit_hi, ls.lit_index + 1);
            return true;
        });
        blob_off += lens[i];
    }
    const size_t ob = align_up(ops.size() * sizeof(ScatterOp), 256), bb = align_up(total + 16, 256);
    const size_t lb = lit_lo < lit_hi ? (size_t)(lit_hi - lit_lo) * 32 : 0;
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(ob + bb + lb + 256));
    if (!h) return LHB200_ENOMEM;
    if (!ops.empty()) {
        uint8_t* d = static_cast<uint8_t*>(dev_scratch(ob + bb));
        if (!d) return LHB200_ENOMEM;
        memcpy(h, ops.data(), ops.size() * sizeof(ScatterOp));
        memcpy(h + ob, data, total);
        LHB_CUDA(cudaMemcpyAsync(d, h, ob + total, cudaMemcpyHostToDevice, c.stream));
        k_scatter_bytes<<<(unsigned)ceil_div(ops.size(), 8), 256, 0, c.stream>>>(reinterpret_cast<const ScatterOp*>(d),
                                                                                 (uint32_t)ops.size(), d + ob);
        count_launch();
        LHB_CUDA(cudaGetLastError());
    }
    if (lb) {
        memcpy(h + ob + bb, &pl.lit[(size_t)lit_lo * 32], lb);
        LHB_CUDA(cudaMemcpyAsync(pl.arena + pl.lit_off + (size_t)lit_lo * 32, h + ob + bb, lb, cudaMemcpyHostToDevice, c.stream));
    }
    LHB_CUDA(cudaStreamSynchronize(c.stream));   // the staging slabs are reused by the next call
    return LHB200_OK;
}
int32_t lhb200_state_patch(lhb200_state* st, uint64_t ssz_offset, const uint8_t* data, uint64_t len) {
    if (len > 0xffffffffull) { set_error("state_patch: a single patch is limited to 4 GiB"); return LHB200_EINVAL; }
    const uint32_t l32 = (uint32_t)len;
    return lhb200_state_patch_batch(st, &ssz_offset, &l32, data, len ? 1 : 0);
}

// (Re)build every level of one resident tree from its leaf chunks.
static void tree_build_levels(lhb200_state::Tree& t, cudaStream_t s) {
    uint64_t n = t.dev.n_leaves;
    for (uint32_t l = 0; l < t.dev.top; l++) {
        k_tree_level<<<(unsigned)ceil_div(ceil_div(n, 2), 256), 256, 0, s>>>(t.dev.lvl[l], n, t.dev.lvl[l + 1], l);
        count_launch();
        n = ceil_div(n, 2);
    }
}
// (Re)build every level of every resident tree from its leaf chunks (which a cold root has just refreshed).
static int32_t state_build_levels(lhb200_state* st, cudaStream_t s) {
    for (lhb200_state::Tree& t : st->trees) {
        tree_build_levels(t, s);
        t.dirty.clear();
        std::fill(t.dirty_bits.begin(), t.dirty_bits.end(), 0ull);
        t.n_marks = 0;
    }
    st->need_full = false;
    LHB_CUDA(cudaGetLastError());
    return LHB200_OK;
}

// Leaf roots of the resizable lists of records and validators, from their items at the current lengths.
static void lists_enqueue_leaves(lhb200_state* st, cudaStream_t s, cudaEvent_t e0, cudaEvent_t e1) {
    for (const lhb200_state::List& L : st->lists) {
        const TreeDev& d = st->trees[L.tree].dev;
        if (d.n_leaves && d.kind != TREE_CHUNKS) enqueue_leaf_roots(d.kind, d.src, d.n_leaves, d.lvl[0], s, e0, e1);
    }
}
// Upload the TreeDev table (through the pinned `h`) and run the finishing step of the lists in `fin`.
static int32_t lists_enqueue_finish(lhb200_state* st, const FinishTable& fin, cudaStream_t s) {
    if (fin.n == 0) return LHB200_OK;
    k_list_finish<<<1, 32, 0, s>>>(st->d_trees, fin);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    for (lhb200_state::List& L : st->lists) L.resized = false;
    return LHB200_OK;
}
static uint64_t finish_units(const TreeDev& d) { return (d.n_leaves ? d.limit_depth - d.top : 0) + 1; }

// Cold root: the plan body, every level of the resident trees (incremental handles), then the tail.  A converted
// handle's plan no longer describes its resizable lists (their leaf launches, reduce passes, ladders and mix-ins
// carried the stage-time lengths and were dropped at conversion): their leaf roots come first, from the resident items
// at the current lengths, and the finishing step writes their field roots before the tail.
static int32_t state_cold_enqueue(lhb200_state* st, cudaStream_t s) {
    lists_enqueue_leaves(st, s, st->e_k0, st->e_k1);
    plan_enqueue_body(st->plan, s, st->e_k0, st->e_k1);
    int32_t rc = state_build_levels(st, s);
    if (rc) return rc;
    if (st->converted) {
        const size_t tb = st->trees.size() * sizeof(TreeDev);
        uint8_t* h = static_cast<uint8_t*>(pinned_scratch(tb));
        if (!h) return LHB200_ENOMEM;
        FinishTable fin{};
        for (size_t k = 0; k < st->trees.size(); k++) {
            lhb200_state::Tree& t = st->trees[k];
            t.dev.dirty = st->d_dirty;
            t.dev.n_dirty = 0;
            memcpy(h + k * sizeof(TreeDev), &t.dev, sizeof(TreeDev));
            if (t.list >= 0) fin.tree[fin.n++] = (uint32_t)k;
        }
        LHB_CUDA(cudaMemcpyAsync(st->d_trees, h, tb, cudaMemcpyHostToDevice, s));
        rc = lists_enqueue_finish(st, fin, s);
        if (rc) return rc;
    }
    st->last_root_hashes = st->plan.hash_units;
    return plan_enqueue_tail(st->plan, s);
}

// Warm root: re-hash the paths above the dirty leaves (one CTA per tree), finish the resizable lists that changed,
// then the tail program.
static int32_t state_incremental_enqueue(lhb200_state* st, cudaStream_t s) {
    uint32_t total = 0;
    for (lhb200_state::Tree& t : st->trees) {
        t.dirty.clear();
        if (t.n_marks) {
            for (size_t w = 0; w < t.dirty_bits.size(); w++) {
                uint64_t bits = t.dirty_bits[w];
                while (bits) {
                    const uint64_t leaf = w * 64 + (uint32_t)__builtin_ctzll(bits);
                    if (leaf < t.dev.n_leaves) t.dirty.push_back((uint32_t)leaf);   // past a truncation: gone
                    bits &= bits - 1;
                }
                t.dirty_bits[w] = 0;
            }
            t.n_marks = 0;
        }
        if (t.dirty.size() > lhb200_state::DIRTY_CAP) {   // too many distinct leaves for the warm buffers: cold root instead
            st->need_full = true;
            return 1;   // (positive: not an error) the caller falls back to the cold path, which also rebuilds the levels
        }
        total += (uint32_t)t.dirty.size();
    }
    uint64_t hashes = st->plan.ops.size();
    FinishTable fin{};
    for (size_t k = 0; k < st->trees.size(); k++) {
        const lhb200_state::Tree& t = st->trees[k];
        if (t.list >= 0 && (!t.dirty.empty() || st->lists[t.list].resized)) {
            fin.tree[fin.n++] = (uint32_t)k;
            hashes += finish_units(t.dev);
        }
    }
    if (total || fin.n) {
        const size_t tb = st->trees.size() * sizeof(TreeDev);
        uint8_t* h = static_cast<uint8_t*>(pinned_scratch(tb + (size_t)total * 4 + 256));
        if (!h) return LHB200_ENOMEM;
        uint32_t* hd = reinterpret_cast<uint32_t*>(h + align_up(tb, 256));
        uint32_t off = 0;
        for (size_t k = 0; k < st->trees.size(); k++) {
            lhb200_state::Tree& t = st->trees[k];
            t.dev.dirty = st->d_dirty + off;
            t.dev.n_dirty = (uint32_t)t.dirty.size();
            if (!t.dirty.empty()) memcpy(hd + off, t.dirty.data(), t.dirty.size() * 4);
            off += t.dev.n_dirty;
            memcpy(h + k * sizeof(TreeDev), &t.dev, sizeof(TreeDev));
            // hashes = distinct parents per level (+ the leaf roots of dirty records): neighbours d[j-1] < d[j] have
            // distinct ancestors exactly at the levels up to the highest bit in which they differ
            if (!t.dirty.empty()) {
                uint64_t cnt = t.dev.top;  // the path of the first dirty leaf
                for (size_t j = 1; j < t.dirty.size(); j++) {
                    const uint32_t hb = 32 - (uint32_t)__builtin_clz(t.dirty[j] ^ t.dirty[j - 1]);  // ancestors equal from level hb up
                    cnt += std::min<uint32_t>(hb - 1, t.dev.top);
                }
                hashes += cnt + (uint64_t)t.leaf.units * t.dirty.size();
            }
            t.dirty.clear();
        }
        LHB_CUDA(cudaMemcpyAsync(st->d_trees, h, tb, cudaMemcpyHostToDevice, s));
        if (total) LHB_CUDA(cudaMemcpyAsync(st->d_dirty, hd, (size_t)total * 4, cudaMemcpyHostToDevice, s));
        // one launch per level covers every tree (blockIdx.y); levels are ordered by the stream
        uint32_t max_nd = 0, max_top = 0;
        bool any_leaf_roots = false;
        for (const lhb200_state::Tree& t : st->trees) {
            max_nd = std::max(max_nd, t.dev.n_dirty);
            if (t.dev.n_dirty) { max_top = std::max(max_top, t.dev.top); any_leaf_roots |= t.dev.kind != TREE_CHUNKS; }
        }
        if (total) {
            const dim3 grid((unsigned)ceil_div(max_nd, 256), (unsigned)st->trees.size());
            for (int l = any_leaf_roots ? -1 : 0; l < (int)max_top; l++) {
                k_tree_update_level<<<grid, 256, 0, s>>>(st->d_trees, l);
                count_launch();
            }
        }
        const int32_t rc = lists_enqueue_finish(st, fin, s);
        if (rc) return rc;
    }
    st->last_root_hashes = hashes;
    return plan_enqueue_tail(st->plan, s);
}

// Switch a resident (unsharded) state to the warm path: allocate and build the level arrays of its big lists
// (validators, balances, inactivity scores, participation x2, randao mixes, block/state roots, slashings).
// Afterwards lhb200_state_patch marks dirty leaves and lhb200_state_root re-hashes only the paths above them
// (plus the tail program); patches outside those lists, or more than 65 536 dirty leaves, fall back to a cold root.
int32_t lhb200_state_enable_incremental(lhb200_state* st) {
    LHB_REQUIRE_READY();
    if (!st) return LHB200_EINVAL;
    if (st->shard.world != 1) { set_error("incremental roots need the whole state on this handle (world == 1)"); return LHB200_EINVAL; }
    if (st->incremental) return LHB200_OK;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    size_t bytes = 0;
    for (const Plan::TreeSpec& ts : st->plan.trees)
        for (uint64_t n = ceil_div(ts.n_chunks, 2);; n = ceil_div(n, 2)) { bytes += align_up(n * 32, 256); if (n == 1) break; }
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_levels), bytes + 256));
    st->levels_bytes = bytes + 256;
    size_t off = 0;
    for (const Plan::TreeSpec& ts : st->plan.trees) {
        lhb200_state::Tree t;
        memset(&t.dev, 0, sizeof t.dev);
        t.dev.src = ts.src;
        t.dev.kind = ts.leaf.tree;
        t.dev.n_leaves = ts.n_chunks;
        t.dev.top = ceil_log2(ts.n_chunks);
        t.dev.top_dst = reinterpret_cast<uint8_t*>(ts.top_addr);
        t.dev.lvl[0] = const_cast<uint8_t*>(ts.chunks);
        uint64_t n = ts.n_chunks;
        for (uint32_t l = 1; l <= t.dev.top; l++) {
            n = ceil_div(n, 2);
            t.dev.lvl[l] = st->d_levels + off;
            off += align_up(n * 32, 256);
        }
        t.leaf = ts.leaf; t.copy = ts.copy; t.item_bytes = ts.item_bytes;
        t.dirty_bits.assign((ts.n_chunks + 63) / 64, 0ull);
        st->trees.push_back(t);
    }
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_trees), st->trees_bytes()));
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_dirty), st->dirty_bytes()));
    index_resident(st);
    st->incremental = true;
    st->need_full = true;   // the first root after enabling is cold and builds the levels
    return LHB200_OK;
}
uint64_t lhb200_state_last_root_hashes(const lhb200_state* st) { return st ? st->last_root_hashes : 0; }

// ---------------------------------------------------------------------------------------------------------
// Resizable lists (lhb200_state_list_edit, lhb200_state_set_payload_header).  A handle keeps its stage-time plan until
// the first such call; then each list of LIST_SPECS moves to storage of its own with headroom (items, leaf
// chunks, every level), its leaf launches and reduce passes leave the cold plan, and its zero ladder and length mix-in
// leave the tail program: k_list_finish writes the field root from the list's current top and length instead.

// LIST_SPECS index of the resizable list `field` of the handle's fork, or -1
static int list_spec_of(const lhb200_state* st, uint32_t field) {
    const int n_fields = fork_layout(st->shard.fork)->state_fields;
    for (int k = 0; k < N_LIST_SPECS; k++)
        if (LIST_SPECS[k].field == field && (int)field < n_fields) return k;
    return -1;
}
static lhb200_state::List& list_of(lhb200_state* st, int spec) {
    for (lhb200_state::List& L : st->lists)
        if (L.spec == spec) return L;
    return st->lists.front();   // not reached: a converted handle has every list of its fork
}
// Hash units the describer counts for a list of `len` items: leaf roots, data tree, zero ladder, length mix-in.
static uint64_t list_units(const ListSpec& sp, uint64_t len) {
    const uint64_t n = list_leaves(sp, len);
    uint64_t u = (uint64_t)sp.leaf.units * len + 1;
    if (n) {
        const uint32_t top = ceil_log2(n);
        u += sp.depth - top;
        for (uint32_t l = 1; l <= top; l++) u += ceil_div(n, 1ull << l);
    }
    return u;
}
// Lay out the storage of a list of `cap` items at `base` (0: size only): items, leaf chunks (validators and records;
// packed lists are their own chunks), then one array per level.  Returns the bytes.
static size_t list_place(TreeDev& d, const ListSpec& sp, uintptr_t base, uint64_t cap) {
    const uint64_t leaves = std::max<uint64_t>(list_leaves(sp, cap), 1);
    size_t off = align_up(cap * sp.item_bytes + 32, 256);
    d.src = reinterpret_cast<const uint8_t*>(base);
    if (sp.leaf.tree == TREE_CHUNKS) {
        d.lvl[0] = reinterpret_cast<uint8_t*>(base);
    } else {
        d.lvl[0] = reinterpret_cast<uint8_t*>(base + off);
        off += align_up(leaves * 32, 256);
    }
    uint64_t n = leaves;
    for (uint32_t l = 1; l <= ceil_log2(leaves); l++) {
        n = ceil_div(n, 2);
        d.lvl[l] = reinterpret_cast<uint8_t*>(base + off);
        off += align_up(n * 32, 256);
    }
    return off;
}
// (Re)allocate a list's storage for `cap` items.  Growth copies the items, leaf chunks and levels device to device.
static int32_t list_alloc(lhb200_state* st, lhb200_state::List& L, uint64_t cap, cudaStream_t s) {
    const ListSpec& sp = LIST_SPECS[L.spec];
    lhb200_state::Tree& t = st->trees[L.tree];
    TreeDev d = t.dev;
    uint8_t* mem = nullptr;
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&mem), list_place(d, sp, 0, cap)));
    list_place(d, sp, reinterpret_cast<uintptr_t>(mem), cap);
    if (L.d_mem) {
        const uint64_t n = t.dev.n_leaves;
        const uint64_t item_bytes = sp.leaf.tree == TREE_CHUNKS ? n * 32 : t.dev.length * sp.item_bytes;   // with the zero pad
        if (item_bytes) LHB_CUDA(cudaMemcpyAsync(mem, L.d_mem, item_bytes, cudaMemcpyDeviceToDevice, s));
        if (sp.leaf.tree != TREE_CHUNKS && n) LHB_CUDA(cudaMemcpyAsync(d.lvl[0], t.dev.lvl[0], n * 32, cudaMemcpyDeviceToDevice, s));
        uint64_t m = n;
        for (uint32_t l = 1; l <= t.dev.top; l++) {
            m = ceil_div(m, 2);
            LHB_CUDA(cudaMemcpyAsync(d.lvl[l], t.dev.lvl[l], m * 32, cudaMemcpyDeviceToDevice, s));
        }
        LHB_CUDA(cudaStreamSynchronize(s));
        LHB_CUDA(cudaFree(L.d_mem));
    }
    L.d_mem = mem;
    L.cap = cap;
    t.dev = d;
    t.dirty_bits.resize(ceil_div(std::max<uint64_t>(list_leaves(sp, cap), 1), 64), 0ull);
    return LHB200_OK;
}

// SSZ offsets of the variable-size fields of the current encoding follow from their lengths: move the lists' resident
// copies, the payload header's literal sources and the hash-unit count along, and rebuild the patch lookups.
static void state_relayout(lhb200_state* st) {
    using namespace state_layout;
    uint64_t off[N_VAR];
    off[0] = fork_layout(st->shard.fork)->state_fixed;
    for (int k = 1; k < N_VAR; k++) off[k] = off[k - 1] + st->var_len[k - 1];
    uint64_t units = st->units_base;
    for (const lhb200_state::List& L : st->lists) {
        const ListSpec& sp = LIST_SPECS[L.spec];
        const lhb200_state::Tree& t = st->trees[L.tree];
        st->copies[t.copy] = {off[sp.var], t.dev.length * sp.item_bytes, L.d_mem, 0};
        units += list_units(sp, t.dev.length);
    }
    st->plan.hash_units = units;
    for (const auto& h : st->hdr_lits) st->plan.lit_src[h.first].src_off = off[V_LEPH] + h.second;
    index_resident(st);
}

// Convert an incremental handle to resizable lists (see LIST_SPECS).  Each list's share of the stage-time plan (leaf
// launches, reduce passes, tail ops and tree; st->marks) is dropped, and its staged copy moves to storage of its own,
// where its tree is built on the device.
static int32_t state_convert(lhb200_state* st, cudaStream_t s) {
    const ForkLayout& fl = *fork_layout(st->shard.fork);
    Plan& pl = st->plan;
    auto cut = [](auto& v, size_t lo, size_t hi) { v.erase(v.begin() + lo, v.begin() + hi); };
    uint64_t stage_units = 0;
    for (int k = N_LIST_SPECS - 1; k >= 0; k--) {   // the last field first: earlier fields' marks stay valid
        const ListSpec& sp = LIST_SPECS[k];
        if ((int)sp.field >= fl.state_fields) continue;
        const PlanMark &a = st->marks[sp.field], &b = st->marks[sp.field + 1];
        cut(pl.leaves, a.leaves, b.leaves);
        for (size_t q = 0; q < pl.passes.size(); q++) cut(pl.passes[q], a.pass(q), b.pass(q));
        cut(pl.ops, a.ops, b.ops);
        cut(pl.op_wave, a.ops, b.ops);
        cut(st->trees, a.trees, b.trees);
        cut(pl.merkle_lists, a.merkle_lists, b.merkle_lists);
        stage_units += list_units(sp, st->var_len[sp.var] / sp.item_bytes);
    }
    pl.passes.erase(std::remove_if(pl.passes.begin(), pl.passes.end(), [](const std::vector<MerkleSeg>& p) { return p.empty(); }),
                    pl.passes.end());
    {   // the pruned tail goes where the stage-time one was (it is shorter)
        const size_t nb = align_up(pl.ops.size() * sizeof(HashOp), 256);
        uint8_t* h = static_cast<uint8_t*>(pinned_scratch(nb + (pl.ops.size() + 2) * 4));
        if (!h) return LHB200_ENOMEM;
        plan_sort_ops(pl, reinterpret_cast<HashOp*>(h));
        memcpy(h + nb, pl.h_waves.data(), pl.h_waves.size() * 4);
        LHB_CUDA(cudaMemcpyAsync(pl.d_ops, h, pl.ops.size() * sizeof(HashOp), cudaMemcpyHostToDevice, s));
        LHB_CUDA(cudaMemcpyAsync(pl.d_waves, h + nb, pl.h_waves.size() * 4, cudaMemcpyHostToDevice, s));
    }
    st->units_base = pl.hash_units - stage_units;
    // every list gets a resizable tree, seeded from the list's one staged copy, which then addresses its storage
    for (int k = 0; k < N_LIST_SPECS; k++) {
        const ListSpec& sp = LIST_SPECS[k];
        if ((int)sp.field >= fl.state_fields) continue;
        const uint64_t len = st->var_len[sp.var] / sp.item_bytes;
        const bool packed = sp.leaf.tree == TREE_CHUNKS;
        lhb200_state::Tree t;
        memset(&t.dev, 0, sizeof t.dev);
        t.dev.kind = sp.leaf.tree;
        t.dev.n_leaves = list_leaves(sp, len);
        t.dev.top = ceil_log2(t.dev.n_leaves);
        t.dev.limit_depth = sp.depth;
        t.dev.length = len;
        t.dev.field_dst = reinterpret_cast<uint8_t*>(st->field_ops[sp.field]);
        t.leaf = sp.leaf;
        t.copy = st->marks[sp.field].copies;
        t.item_bytes = packed ? 32 : sp.item_bytes;
        t.list = (int)st->lists.size();
        const StageCopy staged = st->copies[t.copy];   // zero-padded past its bytes
        st->trees.push_back(std::move(t));
        lhb200_state::List L;
        L.spec = k;
        L.tree = (int)st->trees.size() - 1;
        L.resized = true;
        st->lists.push_back(L);
        int32_t rc = list_alloc(st, st->lists.back(), std::max<uint64_t>(2 * len, 16), s);
        if (rc) return rc;
        const uint64_t nbytes = packed ? 32 * list_leaves(sp, len) : len * sp.item_bytes;
        if (len) LHB_CUDA(cudaMemcpyAsync(st->lists.back().d_mem, staged.dst, nbytes, cudaMemcpyDeviceToDevice, s));
    }
    LHB_CUDA(cudaFree(st->d_trees));
    LHB_CUDA(cudaFree(st->d_dirty));
    st->d_trees = nullptr;
    st->d_dirty = nullptr;
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_trees), st->trees_bytes()));
    LHB_CUDA(cudaMalloc(reinterpret_cast<void**>(&st->d_dirty), st->dirty_bytes()));
    // a tree's dirty pointer only means something between the upload of the tree table and the kernels that read it;
    // the old table is gone, so no tree keeps pointing into it (lhb200_state_clone relocates every address it finds)
    for (lhb200_state::Tree& t : st->trees) {
        t.dev.dirty = nullptr;
        t.dev.n_dirty = 0;
    }
    lists_enqueue_leaves(st, s, nullptr, nullptr);
    for (const lhb200_state::List& L : st->lists) tree_build_levels(st->trees[L.tree], s);
    LHB_CUDA(cudaGetLastError());
    st->converted = true;
    state_relayout(st);
    LHB_CUDA(cudaStreamSynchronize(s));
    return LHB200_OK;
}

static int32_t check_resizable(const lhb200_state* st, const char* what) {
    if (st->shard.world != 1) { set_error("%s: a sharded handle keeps its list lengths", what); return LHB200_EINVAL; }
    if (!st->incremental) { set_error("%s: needs an incremental handle (lhb200_state_enable_incremental)", what); return LHB200_EINVAL; }
    return LHB200_OK;
}

// New length of one list after its items [first, first + n) were written: zero the packed tail, mark the dirty leaves.
static int32_t list_set_length(lhb200_state* st, lhb200_state::List& L, uint64_t new_len, uint64_t first, uint64_t n,
                               cudaStream_t s) {
    const ListSpec& sp = LIST_SPECS[L.spec];
    lhb200_state::Tree& t = st->trees[L.tree];
    const uint64_t old = t.dev.length, nl = list_leaves(sp, new_len), ib = sp.item_bytes;
    if (sp.leaf.tree == TREE_CHUNKS && nl * 32 > new_len * ib)   // SSZ packing pads the last chunk with zeros
        LHB_CUDA(cudaMemsetAsync(L.d_mem + new_len * ib, 0, nl * 32 - new_len * ib, s));
    auto mark = [&](uint64_t a, uint64_t b) {
        if (st->need_full || a >= b) return;
        if (t.n_marks + (b - a) > 4ull * lhb200_state::DIRTY_CAP) { st->need_full = true; return; }
        for (uint64_t q = a; q < b; q++) t.mark(q);
    };
    if (n) mark(sp.leaf.tree == TREE_CHUNKS ? first * ib / 32 : first, list_leaves(sp, first + n));
    if (new_len < old && nl) mark(nl - 1, nl);   // the new right edge: its path re-hashes with zero siblings
    L.resized |= new_len != old;
    t.dev.n_leaves = nl;
    t.dev.top = ceil_log2(nl);
    t.dev.length = new_len;
    st->var_len[sp.var] = new_len * ib;
    return LHB200_OK;
}

int32_t lhb200_state_list_edit(lhb200_state* st, const lhb200_list_edit* edits, uint32_t n_edits, const uint8_t* data) {
    LHB_REQUIRE_READY();
    if (!st || (n_edits && !edits)) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    int32_t rc = check_resizable(st, "state_list_edit");
    if (rc) return rc;
    // every edit is checked before anything changes: a refused call leaves the handle as it was
    uint64_t seen = 0, total = 0;
    for (uint32_t i = 0; i < n_edits; i++) {
        const lhb200_list_edit& e = edits[i];
        const int k = list_spec_of(st, e.field);
        if (k < 0 || e.reserved) {
            set_error("state_list_edit: field %u is not a resizable list of this fork, or reserved != 0", e.field);
            return LHB200_EINVAL;
        }
        if ((seen >> e.field) & 1) { set_error("state_list_edit: two edits of field %u in one call", e.field); return LHB200_EINVAL; }
        seen |= 1ull << e.field;
        const ListSpec& sp = LIST_SPECS[k];
        const uint64_t old = st->var_len[sp.var] / sp.item_bytes;
        if (e.new_len > sp.limit || e.first > e.new_len || e.n > e.new_len - e.first) {
            set_error("state_list_edit: field %u: new_len %llu (limit %llu), first %llu, n %llu", e.field,
                      (unsigned long long)e.new_len, (unsigned long long)sp.limit, (unsigned long long)e.first,
                      (unsigned long long)e.n);
            return LHB200_EINVAL;
        }
        if (e.new_len > old && (e.first > old || e.first + e.n < e.new_len)) {
            set_error("state_list_edit: field %u grows from %llu to %llu items: all new items must be written", e.field,
                      (unsigned long long)old, (unsigned long long)e.new_len);
            return LHB200_EINVAL;
        }
        total += e.n * sp.item_bytes;
    }
    if (total && !data) return LHB200_EINVAL;
    if (n_edits == 0) return LHB200_OK;
    if (!st->converted && (rc = state_convert(st, c.stream))) return rc;
    for (uint32_t i = 0; i < n_edits; i++) {   // capacity first (doubling), device to device
        lhb200_state::List& L = list_of(st, list_spec_of(st, edits[i].field));
        if (edits[i].new_len > L.cap && (rc = list_alloc(st, L, std::max(edits[i].new_len, 2 * L.cap), c.stream))) return rc;
    }
    uint8_t* h = total ? static_cast<uint8_t*>(pinned_scratch(total)) : nullptr;
    if (total && !h) return LHB200_ENOMEM;
    if (total) memcpy(h, data, total);
    uint64_t off = 0;
    for (uint32_t i = 0; i < n_edits; i++) {
        const lhb200_list_edit& e = edits[i];
        lhb200_state::List& L = list_of(st, list_spec_of(st, e.field));
        const uint64_t ib = LIST_SPECS[L.spec].item_bytes;
        if (e.n) LHB_CUDA(cudaMemcpyAsync(L.d_mem + e.first * ib, h + off, e.n * ib, cudaMemcpyHostToDevice, c.stream));
        off += e.n * ib;
        if ((rc = list_set_length(st, L, e.new_len, e.first, e.n, c.stream))) return rc;
    }
    state_relayout(st);
    LHB_CUDA(cudaStreamSynchronize(c.stream));   // the staging slab is reused by the next call
    return LHB200_OK;
}

int32_t lhb200_state_list_len(const lhb200_state* st, uint32_t field, uint64_t* len) {
    LHB_REQUIRE_READY();
    if (!st || !len) return LHB200_EINVAL;
    const int k = list_spec_of(st, field);
    if (k < 0) { set_error("state_list_len: field %u is not a resizable list of this fork", field); return LHB200_EINVAL; }
    *len = st->var_len[LIST_SPECS[k].var] / LIST_SPECS[k].item_bytes;
    return LHB200_OK;
}

// The header hashes the same way whatever extra_data's length (one literal chunk and one length literal), so a
// replacement rewrites literal chunks and moves the offsets of the variable-size fields after it.
int32_t lhb200_state_set_payload_header(lhb200_state* st, const uint8_t* ssz, uint64_t len) {
    LHB_REQUIRE_READY();
    if (!st || (len && !ssz)) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    int32_t rc = check_resizable(st, "state_set_payload_header");
    if (rc) return rc;
    const ForkLayout& fl = *fork_layout(st->shard.fork);
    if (!fl.payload_fields) { set_error("state_set_payload_header: this fork has no execution payload header"); return LHB200_EINVAL; }
    Span v[1];
    if (!read_offsets(ssz, len, fl.header_fixed, block_layout::HEADER_VAR_POS, v) || !v[0].fits(1, 32)) {
        set_error("state_set_payload_header: malformed ExecutionPayloadHeader SSZ (%llu bytes)", (unsigned long long)len);
        return LHB200_EINVAL;
    }
    if (!st->converted && (rc = state_convert(st, c.stream))) return rc;
    Plan& pl = st->plan;
    uint32_t lo = st->hdr_len_chunk, hi = st->hdr_len_chunk + 1;
    for (const auto& hl : st->hdr_lits) {
        Plan::LitSrc& ls = pl.lit_src[hl.first];
        if ((int)hl.first == st->hdr_extra) ls.n = (uint32_t)v[0].len;
        uint8_t* chunk = &pl.lit[(size_t)ls.lit_index * 32];
        memset(chunk, 0, 32);
        memcpy(chunk, ssz + hl.second, ls.n);
        lo = std::min(lo, ls.lit_index);
        hi = std::max(hi, ls.lit_index + 1);
    }
    uint8_t* lc = &pl.lit[(size_t)st->hdr_len_chunk * 32];
    memset(lc, 0, 32);
    for (int k = 0; k < 8; k++) lc[k] = (uint8_t)(v[0].len >> (8 * k));
    const size_t lb = (size_t)(hi - lo) * 32;
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(lb));
    if (!h) return LHB200_ENOMEM;
    memcpy(h, &pl.lit[(size_t)lo * 32], lb);
    LHB_CUDA(cudaMemcpyAsync(pl.arena + pl.lit_off + (size_t)lo * 32, h, lb, cudaMemcpyHostToDevice, c.stream));
    st->var_len[state_layout::V_LEPH] = len;
    state_relayout(st);
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    return LHB200_OK;
}

int32_t lhb200_state_root_enqueue(lhb200_state* st, void* stream, const void** d_root) {
    LHB_REQUIRE_READY();
    if (!st) return LHB200_EINVAL;
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx().stream;
    if (!st->e_k0) { cudaEventCreate(&st->e_k0); cudaEventCreate(&st->e_k1); }
    int32_t rc = 1;
    if (st->incremental && !st->need_full) rc = state_incremental_enqueue(st, s);
    if (rc > 0) rc = state_cold_enqueue(st, s);
    if (rc) return rc;
    rc = gather_operands(st->d_gather, 1 + MAX_FIELDS, st->d_result, s);
    if (rc) return rc;
    if (d_root) *d_root = st->d_result;
    return LHB200_OK;
}

int32_t lhb200_state_root(lhb200_state* st, uint8_t out[32], uint8_t* field_roots) {
    LHB_REQUIRE_READY();
    if (!st || !out) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    int32_t rc = lhb200_state_root_enqueue(st, c.stream, nullptr);
    if (rc) return rc;
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch((1 + MAX_FIELDS) * 32));
    if (!h) return LHB200_ENOMEM;
    LHB_CUDA(cudaMemcpyAsync(h, st->d_result, (1 + MAX_FIELDS) * 32, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out, h, 32);
    // 28 field roots for every fork up to Deneb (the unused tail is zero chunks), 37 for an Electra handle
    if (field_roots) memcpy(field_roots, h + 32, (st->shard.fork == LHB200_FORK_ELECTRA ? MAX_FIELDS : 28) * 32);
    return LHB200_OK;
}

static int32_t proof_events() {
    for (cudaEvent_t& e : g_proof_ev)
        if (!e) LHB_CUDA(cudaEventCreate(&e));
    return LHB200_OK;
}
float lhb200_debug_proof_gather_ms(void) {
    std::lock_guard<std::recursive_mutex> g(ctx().mu);   // the events belong to the calls that record them
    float ms = -1.f;
    if (!g_proof_ev[0] || cudaEventElapsedTime(&ms, g_proof_ev[0], g_proof_ev[1]) != cudaSuccess) { cudaGetLastError(); return -1.f; }
    return ms;
}

// Branches of generalized indices of a resident state.  Every gindex is resolved on the host before the handle is
// touched, so a refused call leaves it as it was; then one root (warm or cold, as lhb200_state_root), the levels the
// proofs rebuild, one gather and one synchronise.
int32_t lhb200_state_proofs(lhb200_state* st, const uint64_t* gindices, uint32_t n, uint8_t* branches, uint8_t root[32]) {
    LHB_REQUIRE_READY();
    if (!st || !root || (n && !gindices)) { set_error("state_proofs: null argument"); return LHB200_EINVAL; }
    if (st->shard.world != 1) { set_error("state_proofs: a sharded handle holds only its share of the lists"); return LHB200_EINVAL; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    ProofResolver pr(st->plan);
    pr.add_state(st);
    int32_t rc;
    for (uint32_t i = 0; i < n; i++)
        if ((rc = pr.resolve(st->root_op, gindices[i]))) return rc;
    const uint64_t total = pr.first.back();
    if (total && !branches) { set_error("state_proofs: null branches"); return LHB200_EINVAL; }
    if ((rc = proof_events())) return rc;
    // pinned: the front is what a root stages (its tree and dirty tables), then the proof tables and the root
    const size_t front = align_up(st->trees_bytes() + st->dirty_bytes(), 256), tb = pr.table_bytes();
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(front + tb + 256));
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(pr.device_bytes()));
    if (!h || !d) return LHB200_ENOMEM;
    if ((rc = pr.upload(h + front, d, c.stream))) return rc;
    if ((rc = lhb200_state_root_enqueue(st, c.stream, nullptr))) return rc;
    if ((rc = pr.enqueue(c.stream, g_proof_ev[0], g_proof_ev[1]))) return rc;
    LHB_CUDA(cudaMemcpyAsync(h + front + tb, st->d_result, 32, cudaMemcpyDeviceToHost, c.stream));
    if (total) LHB_CUDA(cudaMemcpyAsync(branches, pr.d_branches, total * 32, cudaMemcpyDefault, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(root, h + front + tb, 32);
    return LHB200_OK;
}

int32_t lhb200_state_release(lhb200_state* st) {
    if (!st) return LHB200_OK;
    std::lock_guard<std::recursive_mutex> g(ctx().mu);
    if (ctx().ready) cudaStreamSynchronize(ctx().stream);
    if (st->arena) {  // keep one arena around for the next stage call (host-buffer entry point re-stages every call)
        if (g_spare_arena) cudaFree(g_spare_arena);
        g_spare_arena = st->arena;
        g_spare_bytes = st->arena_bytes;
    }
    if (st->e_k0) cudaEventDestroy(st->e_k0);
    if (st->e_k1) cudaEventDestroy(st->e_k1);
    if (st->d_levels) cudaFree(st->d_levels);
    if (st->d_trees) cudaFree(st->d_trees);
    if (st->d_dirty) cudaFree(st->d_dirty);
    if (st->d_coll) cudaFree(st->d_coll);
    for (const lhb200_state::List& L : st->lists) cudaFree(L.d_mem);
    delete st;
    return LHB200_OK;
}

uint64_t lhb200_state_hash_units(const lhb200_state* st) { return st ? st->plan.hash_units : 0; }

// ---------------------------------------------------------------------------------------------------------
// Branches (lhb200_state_clone).  A handle holds absolute device addresses in its plan, its tables and its trees; a
// clone copies the live bytes of every allocation into allocations of its own and rewrites each address through a map
// from the source's allocations to the clone's.
}  // extern "C"
namespace lhb200 {
// Every device address a handle holds, as f(address, bytes): bytes > 0 for the base of an allocation the handle owns
// (the arena first), 0 for an address into one.  Null addresses and zero-hash operands (OP_ZERO_FLAG) are passed too.
// f may rewrite the address.  The clone and lhb200_debug_state_disjoint both walk a handle through this one function.
template <class F>
static void visit_device_addresses(lhb200_state* st, F&& f) {
    auto at = [&](auto*& p, size_t bytes = 0) {
        uint64_t a = reinterpret_cast<uint64_t>(p);
        f(a, bytes);
        p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(a);
    };
    at(st->arena, st->arena_bytes);
    if (st->d_levels) at(st->d_levels, st->levels_bytes);
    if (st->d_trees) at(st->d_trees, st->trees_bytes());
    if (st->d_dirty) at(st->d_dirty, st->dirty_bytes());
    if (st->d_coll) at(st->d_coll, st->coll_bytes());
    for (lhb200_state::List& L : st->lists) {
        TreeDev d;
        at(L.d_mem, list_place(d, LIST_SPECS[L.spec], 0, L.cap));
    }
    Plan& pl = st->plan;
    at(pl.arena);
    for (LeafLaunch& L : pl.leaves) { at(L.in); at(L.out); }
    for (auto& pass : pl.passes)
        for (MerkleSeg& sg : pass) { at(sg.in); at(sg.out); }
    for (HashOp& op : pl.ops) { f(op.dst, 0); f(op.a, 0); f(op.b, 0); }
    for (ByteItem& it : pl.items) { at(it.src); at(it.out); }
    for (Plan::TreeSpec& ts : pl.trees) { at(ts.chunks); f(ts.top_addr, 0); at(ts.src); }
    for (Plan::ListRec& lr : pl.merkle_lists) { at(lr.chunks); f(lr.top_addr, 0); }
    at(pl.d_ops); at(pl.d_waves); at(pl.d_items);
    for (StageCopy& cp : st->copies) at(cp.dst);
    for (uint64_t& op : st->field_ops) f(op, 0);
    f(st->root_op, 0);
    at(st->d_gather); at(st->d_result);
    for (ShardedList& L : st->sharded) f(L.local_op, 0);
    for (lhb200_state::Tree& t : st->trees) {
        at(t.dev.src);
        for (uint8_t*& l : t.dev.lvl) at(l);
        at(t.dev.top_dst); at(t.dev.dirty); at(t.dev.field_dst);
    }
}
static bool is_device_address(uint64_t a) { return a && !(a & OP_ZERO_FLAG); }

// An allocation of a source handle and where the clone's copy of it starts.
struct Relocation {
    uint64_t from, bytes, to;
};
// Sorted by `from`: the address a moves to, or 0 if it lies in no allocation.
static uint64_t relocate(const std::vector<Relocation>& map, uint64_t a) {
    auto r = std::upper_bound(map.begin(), map.end(), a, [](uint64_t x, const Relocation& m) { return x < m.from; });
    if (r == map.begin()) return 0;
    --r;
    return a - r->from < r->bytes ? a - r->from + r->to : 0;
}
// The bytes of a handle that a clone copies, as g(address, bytes), each range rounded up to 16 inside its allocation:
// the arena up to its allocation cursor, the levels, and per resizable list its items, leaf chunks and each level up
// to the current length (list_alloc relies on the same: nothing past the length is read before it is written).
template <class G>
static void visit_live_ranges(const lhb200_state* st, G&& g) {
    auto live = [&](const void* p, uint64_t bytes) {
        if (bytes) g(static_cast<const uint8_t*>(p), align_up(bytes, 16));
    };
    live(st->arena, st->plan.bump);
    live(st->d_levels, st->levels_bytes);
    for (const lhb200_state::List& L : st->lists) {
        const TreeDev& d = st->trees[L.tree].dev;
        if (d.kind != TREE_CHUNKS) live(d.src, d.length * LIST_SPECS[L.spec].item_bytes);
        uint64_t n = d.n_leaves;
        live(d.lvl[0], n * 32);
        for (uint32_t l = 1; l <= d.top; l++) live(d.lvl[l], (n = ceil_div(n, 2)) * 32);
    }
}
}  // namespace lhb200
extern "C" {

int32_t lhb200_state_device_bytes(const lhb200_state* st, uint64_t* bytes) {
    LHB_REQUIRE_READY();
    if (!st || !bytes) return LHB200_EINVAL;
    std::lock_guard<std::recursive_mutex> g(ctx().mu);
    uint64_t sum = 0;
    visit_device_addresses(const_cast<lhb200_state*>(st), [&](uint64_t&, size_t n) { sum += n; });
    *bytes = sum;
    return LHB200_OK;
}

int32_t lhb200_debug_state_live_bytes(const lhb200_state* st, uint64_t* bytes) {
    LHB_REQUIRE_READY();
    if (!st || !bytes) return LHB200_EINVAL;
    std::lock_guard<std::recursive_mutex> g(ctx().mu);
    uint64_t sum = 0;
    visit_live_ranges(st, [&](const uint8_t*, uint64_t n) { sum += n; });
    *bytes = sum;
    return LHB200_OK;
}

int32_t lhb200_debug_state_disjoint(const lhb200_state* a, const lhb200_state* b, int32_t* disjoint) {
    LHB_REQUIRE_READY();
    if (!a || !b || !disjoint) return LHB200_EINVAL;
    std::lock_guard<std::recursive_mutex> g(ctx().mu);
    std::vector<Relocation> allocs;   // b's allocations (`to` unused)
    visit_device_addresses(const_cast<lhb200_state*>(b), [&](uint64_t& p, size_t n) {
        if (n && p) allocs.push_back({p, n, p});
    });
    std::sort(allocs.begin(), allocs.end(), [](const Relocation& x, const Relocation& y) { return x.from < y.from; });
    bool hit = false;
    visit_device_addresses(const_cast<lhb200_state*>(a), [&](uint64_t& p, size_t) {
        hit |= is_device_address(p) && relocate(allocs, p) != 0;
    });
    *disjoint = hit ? 0 : 1;
    return LHB200_OK;
}

int32_t lhb200_state_clone(const lhb200_state* src, lhb200_state** out) {
    LHB_REQUIRE_READY();
    if (!src || !out) return LHB200_EINVAL;
    if (src->shard.world != 1) { set_error("state_clone: a sharded handle cannot be cloned"); return LHB200_EINVAL; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    // The host state as it is (plan, literals, dirty bitmaps, lengths, patch lookups).  Before anything can fail, the
    // copy forgets the source's allocations and events, so that releasing a failed clone frees only its own.
    std::unique_ptr<lhb200_state, int32_t (*)(lhb200_state*)> st(new lhb200_state(*src), lhb200_state_release);
    st->e_k0 = st->e_k1 = nullptr;
    // Allocations of the same sizes as the source's; the arena may be the spare one a released handle left behind.
    std::vector<Relocation> map;
    int32_t rc = LHB200_OK;
    visit_device_addresses(st.get(), [&](uint64_t& p, size_t n) {
        if (!n || !p) return;
        const uint64_t from = p;
        p = 0;
        if (rc) return;
        void* mem = nullptr;
        if (map.empty() && g_spare_arena && g_spare_bytes >= n) {
            mem = g_spare_arena;
            st->arena_bytes = g_spare_bytes;
            g_spare_arena = nullptr;
            g_spare_bytes = 0;
        } else {
            const cudaError_t e = cudaMalloc(&mem, n);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMalloc(state_clone)"); return; }
        }
        p = reinterpret_cast<uint64_t>(mem);
        map.push_back({from, n, p});
    });
    if (rc) return rc;
    std::sort(map.begin(), map.end(), [](const Relocation& x, const Relocation& y) { return x.from < y.from; });
    std::vector<CopyRange> ranges;
    visit_live_ranges(src, [&](const uint8_t* p, uint64_t bytes) {
        ranges.push_back({reinterpret_cast<uint8_t*>(relocate(map, reinterpret_cast<uint64_t>(p))), p, bytes});
    });
    // Every address the clone holds moves into its own allocations; one that lies in none is refused rather than
    // left pointing into the source.
    bool missed = false;
    visit_device_addresses(st.get(), [&](uint64_t& p, size_t n) {
        if (n || !is_device_address(p)) return;
        const uint64_t q = relocate(map, p);
        missed |= q == 0;
        p = q;
    });
    for (const CopyRange& r : ranges) missed |= r.dst == nullptr;
    if (missed) { set_error("internal: state_clone found a device address outside the source's allocations"); return LHB200_EINVAL; }
    // The tables that hold addresses are uploaded again from the relocated host copies: the tail program, the byte
    // items and the gather table.  The tree and dirty tables need nothing: every root uploads them.
    Plan& pl = st->plan;
    std::vector<uint64_t> gather(1, st->root_op);
    gather.insert(gather.end(), st->field_ops, st->field_ops + MAX_FIELDS);
    const size_t n_ranges = ranges.size();
    const size_t rb = align_up(n_ranges * sizeof(CopyRange), 256), wb = align_up((n_ranges + 1) * 8, 256);
    const size_t ob = align_up(pl.ops.size() * sizeof(HashOp), 256), ib = align_up(pl.items.size() * sizeof(ByteItem), 256);
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(rb + wb + ob + ib + gather.size() * sizeof(HashOp)));
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(rb + wb));
    if (!h || !d) return LHB200_ENOMEM;
    memcpy(h, ranges.data(), n_ranges * sizeof(CopyRange));
    uint64_t* word = reinterpret_cast<uint64_t*>(h + rb);
    word[0] = 0;
    for (size_t i = 0; i < n_ranges; i++) word[i + 1] = word[i] + ranges[i].bytes / 16;
    LHB_CUDA(cudaMemcpyAsync(d, h, rb + (n_ranges + 1) * 8, cudaMemcpyHostToDevice, c.stream));
    int n_sm = 0;
    LHB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, c.device));
    const unsigned grid = (unsigned)std::min<uint64_t>(ceil_div(word[n_ranges], 256), 8ull * n_sm);
    k_copy_ranges<<<grid, 256, 0, c.stream>>>(reinterpret_cast<const CopyRange*>(d), reinterpret_cast<const uint64_t*>(d + rb),
                                             (uint32_t)n_ranges);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    if (!pl.ops.empty()) {
        plan_sort_ops(pl, reinterpret_cast<HashOp*>(h + rb + wb));
        LHB_CUDA(cudaMemcpyAsync(pl.d_ops, h + rb + wb, pl.ops.size() * sizeof(HashOp), cudaMemcpyHostToDevice, c.stream));
    }
    if (!pl.items.empty()) {
        memcpy(h + rb + wb + ob, pl.items.data(), pl.items.size() * sizeof(ByteItem));
        LHB_CUDA(cudaMemcpyAsync(pl.d_items, h + rb + wb + ob, pl.items.size() * sizeof(ByteItem), cudaMemcpyHostToDevice,
                                 c.stream));
    }
    rc = stage_operands(gather, st->d_gather, h + rb + wb + ob + ib, c.stream);
    if (rc) return rc;
    LHB_CUDA(cudaStreamSynchronize(c.stream));   // the staging slabs are reused by the next call
    *out = st.release();
    return LHB200_OK;
}

float lhb200_state_dominant_kernel_ms(const lhb200_state* st) {
    float ms = -1.f;
    if (!st || !st->e_k0 || cudaEventElapsedTime(&ms, st->e_k0, st->e_k1) != cudaSuccess) { cudaGetLastError(); return -1.f; }
    return ms;
}

int32_t lhb200_beacon_state_root_deneb(const uint8_t* ssz, uint64_t len, uint8_t out[32], uint8_t* field_roots) {
    return lhb200_beacon_state_root(ssz, len, LHB200_FORK_DENEB, out, field_roots);
}
// BeaconState::update_tree_hash_cache for any post-Altair variant of the superstruct (beacon_state.rs:224-571).
// field_roots (optional): 28 x 32 bytes (entries beyond the fork's field count are the zero chunk); 37 x 32 for Electra.
int32_t lhb200_beacon_state_root(const uint8_t* ssz, uint64_t len, int32_t fork, uint8_t out[32], uint8_t* field_roots) {
    LHB_REQUIRE_READY();
    lhb200_state* st = nullptr;
    int32_t rc = lhb200_state_stage(ssz, len, fork, &st);
    if (rc) return rc;
    rc = lhb200_state_root(st, out, field_roots);
    lhb200_state_release(st);
    return rc;
}

int32_t lhb200_merkle_tree_proof(const uint8_t* leaves, uint64_t n, uint32_t depth, uint64_t index, uint8_t root[32],
                                 uint8_t* branch) {
    LHB_REQUIRE_READY();
    if (!root || (depth && !branch) || (n && !leaves) || depth > 32 || n > (1ull << depth) ||
        (depth < 64 && index >= (1ull << depth))) {
        set_error("merkle_tree_proof: bad arguments");
        return LHB200_EINVAL;
    }
    // Level-by-level device build (every level materialised so siblings can be read back), then gather.
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    std::vector<uint64_t> cnt(depth + 1);
    cnt[0] = n;
    size_t total = align_up(std::max<uint64_t>(n, 1) * 32, 256);
    for (uint32_t l = 1; l <= depth; l++) {
        cnt[l] = ceil_div(cnt[l - 1], 2);
        total += align_up(std::max<uint64_t>(cnt[l], 1) * 32, 256);
    }
    size_t gath_bytes = (depth + 1) * sizeof(HashOp);
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(total + gath_bytes + (depth + 1) * 32 + 1024));
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(n * 32 + gath_bytes + (depth + 1) * 32 + 512));
    if (!d || !h) return LHB200_ENOMEM;
    if (n) {
        memcpy(h, leaves, n * 32);
        LHB_CUDA(cudaMemcpyAsync(d, h, n * 32, cudaMemcpyHostToDevice, c.stream));
    }
    std::vector<uint8_t*> lvl(depth + 1);
    size_t off = 0;
    for (uint32_t l = 0; l <= depth; l++) {
        lvl[l] = d + off;
        off += align_up(std::max<uint64_t>(cnt[l], 1) * 32, 256);
    }
    for (uint32_t l = 0; l < depth && cnt[l] > 0; l++) {
        MerkleSegTable tab;
        tab.n = 1;
        tab.s[0].in = lvl[l]; tab.s[0].out = lvl[l + 1]; tab.s[0].n_in = cnt[l]; tab.s[0].level_in = l;
        tab.s[0].tile_log = 1; tab.s[0].cta_begin = 0; tab.s[0].n_tiles = (uint32_t)cnt[l + 1];
        k_merkle_reduce<<<(unsigned)cnt[l + 1], REDUCE_THREADS, 0, c.stream>>>(tab);
        count_launch();
    }
    LHB_CUDA(cudaGetLastError());
    std::vector<uint64_t> ops(depth + 1);
    ops[0] = n ? reinterpret_cast<uint64_t>(lvl[depth]) : (OP_ZERO_FLAG | depth);
    uint64_t idx = index;
    for (uint32_t l = 0; l < depth; l++) {
        uint64_t sib = idx ^ 1;
        ops[l + 1] = sib < cnt[l] ? reinterpret_cast<uint64_t>(lvl[l] + 32 * sib) : (OP_ZERO_FLAG | l);
        idx >>= 1;
    }
    uint8_t* h_g = h + align_up(n * 32, 256);
    uint8_t* d_g = d + total;
    uint8_t* d_res = d_g + align_up(gath_bytes, 256);
    int32_t rc = stage_operands(ops, reinterpret_cast<HashOp*>(d_g), h_g, c.stream);
    if (!rc) rc = gather_operands(reinterpret_cast<HashOp*>(d_g), depth + 1, d_res, c.stream);
    if (rc) return rc;
    uint8_t* h_res = h_g + align_up(gath_bytes, 256);
    LHB_CUDA(cudaMemcpyAsync(h_res, d_res, (depth + 1) * 32, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(root, h_res, 32);
    if (depth) memcpy(branch, h_res + 32, depth * 32);
    return LHB200_OK;
}

int32_t lhb200_verify_merkle_proofs(const uint8_t* leaves, const uint8_t* branches, uint32_t depth,
                                    const uint64_t* indices, const uint8_t* roots, uint64_t n, uint8_t* ok) {
    LHB_REQUIRE_READY();
    if (n == 0) return LHB200_OK;
    if (!leaves || !indices || !roots || !ok || (depth && !branches)) return LHB200_EINVAL;
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    size_t b_leaves = align_up(n * 32, 256), b_br = align_up(n * depth * 32 + 32, 256), b_idx = align_up(n * 8, 256),
           b_roots = align_up(n * 32, 256), b_ok = align_up(n, 256);
    size_t tot = b_leaves + b_br + b_idx + b_roots + b_ok;
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(tot));
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(tot));
    if (!d || !h) return LHB200_ENOMEM;
    memcpy(h, leaves, n * 32);
    if (depth) memcpy(h + b_leaves, branches, n * depth * 32);
    memcpy(h + b_leaves + b_br, indices, n * 8);
    memcpy(h + b_leaves + b_br + b_idx, roots, n * 32);
    LHB_CUDA(cudaMemcpyAsync(d, h, tot - b_ok, cudaMemcpyHostToDevice, c.stream));
    k_verify_branches<<<(unsigned)ceil_div(n, 128), 128, 0, c.stream>>>(
        d, d + b_leaves, depth, reinterpret_cast<const uint64_t*>(d + b_leaves + b_br), d + b_leaves + b_br + b_idx, n,
        d + tot - b_ok);
    count_launch();
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(h + tot - b_ok, d + tot - b_ok, n, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(ok, h + tot - b_ok, n);
    return LHB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// BeaconBlock (mainnet preset) of any fork from Altair to Electra: BeaconBlock::canonical_root
// (consensus/types/src/beacon_block.rs:158-160).  Layouts: beacon_block.rs:41-90, beacon_block_body.rs:43-121,
// execution_payload.rs:54-101, sizes and limits per fork in FORK_LAYOUTS; operation containers as cited in
// include/lhb200.h.  The host only walks SSZ offsets: every packed byte string (transactions, signatures, pubkeys,
// bit lists, index lists, proofs, blooms) is hashed by k_byte_items straight from the staged blob, fixed 8/20/32-byte
// fields become literal chunks, and the container structure above them is a hash program.  The up to 8 192
// DepositRequest records of an Electra payload are the one list of fixed-size containers in a block that can reach
// thousands of items: past 64 records, k_record_roots kind 4 hashes them straight from the staged blob, the reduce
// passes fold them, and the host plans no node per record.
}  // extern "C"
namespace {
struct BlockDescriber : SszDescriber {
    bool blinded = false;   // BlindedBeaconBlock: the body carries an ExecutionPayloadHeader

    uint64_t blob(uint64_t off, uint64_t n, uint32_t depth) { return p.bytes_item(d + off, n, depth, false); }
    uint64_t sig(uint64_t off) { return blob(off, 96, 2); }
    uint64_t pubkey(uint64_t off) { return blob(off, 48, 1); }
    uint64_t att_data(uint64_t off) {  // 128 B (attestation_data.rs:28)
        return p.container({u64(off), u64(off + 8), h256(off + 16), checkpoint(off + 48), checkpoint(off + 88)});
    }
    uint64_t signed_header(uint64_t off) {  // 208 B
        uint64_t h = block_header(off);
        return p.op_hash(h, sig(off + 112));
    }
    uint64_t proposer_slashing(uint64_t off) { return p.op_hash(signed_header(off), signed_header(off + 208)); }
    // IndexedAttestation: attesting_indices (List[u64]) behind a 228-byte fixed part
    uint64_t indexed_attestation(uint64_t off, uint64_t len) {
        Span v[1];
        if (!read_offsets(s + off, len, 228, block_layout::FIRST_VAR_POS, v) || !v[0].fits(8, fl.max_attesting_indices))
            return fail();
        uint64_t idx = p.bytes_item(d + off + v[0].off, v[0].len, packed_depth(8 * fl.max_attesting_indices), true,
                                    v[0].len / 8);
        return p.container({idx, att_data(off + 4), sig(off + 132)});
    }
    // Attestation: aggregation_bits (Bitlist), data, then the signature at the end of the fixed part; Electra puts
    // committee_bits (Bitvector[64]) between data and signature (attestation.rs:76-82)
    uint64_t attestation(uint64_t off, uint64_t len) {
        const uint32_t fixed = fl.attestation_fixed, o_sig = fixed - 96;
        Span v[1];
        if (!read_offsets(s + off, len, fixed, block_layout::FIRST_VAR_POS, v) || v[0].len == 0 || s[off + len - 1] == 0)
            return fail();
        const uint8_t last = s[off + len - 1];
        int top = 7;
        while (!((last >> top) & 1)) top--;
        const uint64_t bitlen = 8 * (v[0].len - 1) + (uint64_t)top;
        if (bitlen > fl.max_aggregation_bits) return fail();
        // drop the delimiter: either the whole last byte (top == 0) or its top bit
        uint64_t bits = p.bytes_item(d + off + fixed, (bitlen + 7) / 8, packed_depth(fl.max_aggregation_bits / 8), true,
                                     bitlen, top ? (uint32_t)((1u << top) - 1) : 0xff);
        const uint64_t data = att_data(off + 4);
        if (o_sig > 132) return p.container({bits, data, u64(off + 132), sig(off + o_sig)});   // + committee_bits
        return p.container({bits, data, sig(off + o_sig)});
    }
    uint64_t deposit(uint64_t off) {  // 1240 B
        uint64_t data = p.container({pubkey(off + 1056), h256(off + 1104), u64(off + 1136), sig(off + 1144)});
        return p.op_hash(blob(off, 33 * 32, 6), data);
    }
    uint64_t voluntary_exit(uint64_t off) { return p.op_hash(p.op_hash(u64(off), u64(off + 8)), sig(off + 16)); }
    uint64_t bls_change(uint64_t off) {
        return p.op_hash(p.container({u64(off), pubkey(off + 8), addr20(off + 56)}), sig(off + 76));
    }
    uint64_t withdrawal(uint64_t off) { return p.container({u64(off), u64(off + 8), addr20(off + 16), u64(off + 36)}); }
    // DepositRequest (deposit_request.rs:23-29): 192 B; k_record_roots kind 4 computes the same root on the device
    static constexpr uint64_t DEPOSIT_REQUESTS_AS_OPS = 64;
    uint64_t deposit_request(uint64_t off) {
        return p.container({pubkey(off), h256(off + 48), u64(off + 80), sig(off + 88), u64(off + 184)});
    }
    // List[DepositRequest, 8192] at span x of the payload at `base`: depth 13.  The record kernel and its reduce pass add
    // two serial launches per block (k_record_roots is one thread's chain of 10 hashes); host planning costs ~0.7 us per
    // record.  On an H100 the ops are faster up to 64 records and the kernel past that (DESIGN §3.5).
    uint64_t deposit_requests(uint64_t base, Span x) {
        const uint64_t n = x.len / 192;
        if (n <= DEPOSIT_REQUESTS_AS_OPS || !x.fits(192, 8192))   // fixed_list refuses a malformed list
            return fixed_list(base, x, 192, 13, [&](uint64_t o) { return deposit_request(o); });
        return p.mix_in_length(p.merkle_list(p.leaf_kernel(LEAF_DEPOSIT_REQUEST, d + base + x.off, n), n, 13), n);
    }
    // ExecutionLayerWithdrawalRequest (execution_layer_withdrawal_request.rs:23-26): 76 B
    uint64_t withdrawal_request(uint64_t off) { return p.container({addr20(off), pubkey(off + 20), u64(off + 68)}); }
    // SignedConsolidation (signed_consolidation.rs:23-24, consolidation.rs:24-27): 120 B
    uint64_t consolidation(uint64_t off) {
        return p.op_hash(p.container({u64(off), u64(off + 8), u64(off + 16)}), sig(off + 24));
    }
    uint64_t list_of(std::vector<uint64_t>& roots, uint32_t limit_log) {
        uint64_t n = roots.size();
        uint64_t r = p.small_tree(roots, std::min<uint32_t>(limit_log, ceil_log2(std::max<uint64_t>(n, 1))));
        if (n == 0) r = Plan::zero_op(limit_log);
        else for (uint32_t l = ceil_log2(n); l < limit_log; l++) r = p.op_hash(r, Plan::zero_op(l));
        return p.mix_in_length(r, n);
    }
    // list of `item`-byte containers at span x of the container at `base`, limit 2^limit_log
    template <class F>
    uint64_t fixed_list(uint64_t base, Span x, uint32_t item, uint32_t limit_log, F&& f) {
        if (!x.fits(item, 1ull << limit_log)) return fail();
        std::vector<uint64_t> roots;
        for (uint64_t i = 0; i < x.len / item; i++) roots.push_back(f(base + x.off + item * i));
        return list_of(roots, limit_log);
    }
    // offsets table of a list of variable-size items occupying [off, off+len)
    bool var_bounds(uint64_t off, uint64_t len, uint64_t max_n, std::vector<uint64_t>& b) {
        b.clear();
        if (len == 0) { b.push_back(0); return true; }
        if (len < 4) return false;
        const uint32_t first = rd32(s + off);
        if (first % 4 || first == 0 || first > len || first / 4 > max_n) return false;
        for (uint32_t i = 0; i < first / 4; i++) b.push_back(rd32(s + off + 4 * i));
        b.push_back(len);
        for (size_t i = 0; i + 1 < b.size(); i++)
            if (b[i] > b[i + 1]) return false;
        return true;
    }
    // ExecutionPayload: the prefix and transactions, then the fields later forks append
    uint64_t payload(uint64_t off, uint64_t len) {
        using namespace block_layout;
        Span v[N_PAYLOAD_VAR];
        if (!read_offsets(s + off, len, fl.payload_fixed, PAYLOAD_VAR_POS, v) || !v[P_EXTRA_DATA].fits(1, 32)) return fail();
        std::vector<uint64_t> f = payload_prefix(off, v[P_EXTRA_DATA]), b, roots;
        const Span tx = v[P_TRANSACTIONS];
        if (!var_bounds(off + tx.off, tx.len, 1u << 20, b)) return fail();
        for (size_t i = 0; i + 1 < b.size(); i++)  // ByteList[2^30]: 2^25 chunks
            roots.push_back(p.bytes_item(d + off + tx.off + b[i], b[i + 1] - b[i], 25, true, b[i + 1] - b[i]));
        f.push_back(list_of(roots, 20));
        for (int k = PAYLOAD_PREFIX_FIELDS + 1; k < fl.payload_fields && !bad; k++) {   // appended by later forks
            switch (k) {
                case 14: f.push_back(fixed_list(off, v[P_WITHDRAWALS], 44, 4, [&](uint64_t o) { return withdrawal(o); })); break;
                case 15: case 16: f.push_back(u64(off + 512 + 8 * (k - 15))); break;   // blob_gas_used, excess_blob_gas
                case 17: f.push_back(deposit_requests(off, v[P_DEPOSIT_REQUESTS])); break;
                default: f.push_back(fixed_list(off, v[P_WITHDRAWAL_REQUESTS], 76, 4, [&](uint64_t o) { return withdrawal_request(o); }));
            }
        }
        return bad ? 0 : p.container(f);
    }
    uint64_t body(uint64_t off, uint64_t len, uint64_t dst) {
        using namespace block_layout;
        Span v[N_BODY_VAR];
        if (!read_offsets(s + off, len, fl.body_fixed, BODY_VAR_POS, v)) return fail();
        std::vector<uint64_t> f(9), b, roots;
        f[0] = sig(off);
        f[1] = eth1_data(off + 96);
        f[2] = h256(off + 168);
        f[3] = fixed_list(off, v[B_PROPOSER_SLASHINGS], 416, 4, [&](uint64_t o) { return proposer_slashing(o); });
        const Span as = v[B_ATTESTER_SLASHINGS], at = v[B_ATTESTATIONS];
        if (!var_bounds(off + as.off, as.len, fl.max_attester_slashings, b)) return fail();
        for (size_t i = 0; i + 1 < b.size(); i++) {   // AttesterSlashing: two IndexedAttestations
            const uint64_t q = off + as.off + b[i];
            Span a[2];
            if (!read_offsets(s + q, b[i + 1] - b[i], 8, ATTESTER_SLASHING_VAR_POS, a)) return fail();
            uint64_t r1 = indexed_attestation(q + a[0].off, a[0].len), r2 = indexed_attestation(q + a[1].off, a[1].len);
            if (bad) return 0;
            roots.push_back(p.op_hash(r1, r2));
        }
        f[4] = list_of(roots, ceil_log2(fl.max_attester_slashings));
        roots.clear();
        if (!var_bounds(off + at.off, at.len, fl.max_attestations, b)) return fail();
        for (size_t i = 0; i + 1 < b.size(); i++) {
            roots.push_back(attestation(off + at.off + b[i], b[i + 1] - b[i]));
            if (bad) return 0;
        }
        f[5] = list_of(roots, ceil_log2(fl.max_attestations));
        f[6] = fixed_list(off, v[B_DEPOSITS], 1240, 4, [&](uint64_t o) { return deposit(o); });
        f[7] = fixed_list(off, v[B_EXITS], 112, 4, [&](uint64_t o) { return voluntary_exit(o); });
        f[8] = p.op_hash(blob(off + 220, 64, 1), sig(off + 284));  // sync_aggregate.rs:38
        for (int k = 9; k < fl.body_fields && !bad; k++) {   // appended by later forks
            const Span x = v[B_PAYLOAD + (k - 9)];
            switch (k) {
                case 9: f.push_back(blinded ? payload_header(off + x.off, x.len) : payload(off + x.off, x.len)); break;
                case 10: f.push_back(fixed_list(off, x, 172, 4, [&](uint64_t o) { return bls_change(o); })); break;
                case 11: f.push_back(fixed_list(off, x, 48, 12, [&](uint64_t o) { return pubkey(o); })); break;  // kzg_commitment.rs:51
                default: f.push_back(fixed_list(off, x, 120, 0, [&](uint64_t o) { return consolidation(o); })); break;  // 12
            }
        }
        if (bad) return 0;
        return p.container(f, dst);
    }
    uint64_t block(uint64_t off, uint64_t len, uint64_t dst_root, uint64_t dst_body) {
        Span v[1];
        if (!read_offsets(s + off, len, block_layout::BLOCK_FIXED, block_layout::BLOCK_VAR_POS, v)) return fail();
        uint64_t b = body(off + v[0].off, v[0].len, dst_body);
        if (bad) return 0;
        return p.container({u64(off), u64(off + 8), h256(off + 16), h256(off + 48), b}, dst_root);
    }
};
}  // namespace
extern "C" {

constexpr int32_t LHB200_ERETRY = -1000;   // internal: the plan did not fit the arena bound of this attempt

// transactions in one BeaconBlock blob (0 when the offsets are not plausible — the describer reports that)
static uint64_t prescan_transactions(const uint8_t* blk, uint64_t len, const ForkLayout& fl) {
    using namespace block_layout;
    Span block[1], body[N_BODY_VAR], pay[N_PAYLOAD_VAR];
    if (!fl.payload_fields || !read_offsets(blk, len, BLOCK_FIXED, BLOCK_VAR_POS, block)) return 0;
    const uint8_t* b = blk + block[0].off;
    if (!read_offsets(b, block[0].len, fl.body_fixed, BODY_VAR_POS, body)) return 0;
    const uint8_t* ep = b + body[B_PAYLOAD].off;
    if (!read_offsets(ep, body[B_PAYLOAD].len, fl.payload_fixed, PAYLOAD_VAR_POS, pay)) return 0;
    const Span tx = pay[P_TRANSACTIONS];
    if (tx.len < 4) return 0;
    const uint64_t first = rd32(ep + tx.off);
    return first <= tx.len ? first / 4 : 0;
}

// Proofs below the body roots of a block batch (lhb200_beacon_block_body_proofs), and the device and pinned bytes
// their tables, rebuilt levels and branches can take.
struct BodyProofs {
    const uint32_t* block_of;
    const uint64_t* gindices;
    uint32_t n;
    uint8_t* branches;
    size_t dev_bytes, host_bytes;
};

static int32_t block_roots_attempt(Ctx& c, const uint8_t* ssz, const uint64_t* offsets, uint32_t n, uint8_t* roots,
                                   uint8_t* body_roots, bool blinded, const ForkLayout& fl, uint64_t base, uint64_t total, size_t in_pad,
                                   size_t max_nodes, size_t lit_cap, const BodyProofs* pq) {
    uint8_t *d_in = nullptr, *d_roots = nullptr, *d_body = nullptr;
    bool bad = false;
    auto build = [&](Plan& p) {
        d_in = p.alloc(in_pad);
        d_roots = p.alloc(64ull * n);
        d_body = d_roots + 32ull * n;
        p.forced_base = reinterpret_cast<uint64_t>(d_roots);
        p.forced_wave.assign(2ull * n, -1);
        BlockDescriber bd{{p, ssz + base, d_in, fl}, blinded};
        for (uint32_t i = 0; i < n && !bd.bad; i++)
            bd.block(offsets[i] - base, offsets[i + 1] - offsets[i], reinterpret_cast<uint64_t>(d_roots + 32ull * i),
                     reinterpret_cast<uint64_t>(d_body + 32ull * i));
        bad = bd.bad;
        return LHB200_OK;
    };
    // One planning pass over the bounded arena (host time matters here: a block is only ~10^4 hashes).
    const size_t prog_bytes = program_bytes(max_nodes, max_nodes);
    // literals | node pool (op outputs) | staged blob | roots | item outputs, leaf-kernel roots and reduce outputs
    // (one 32-byte root per 192-byte DepositRequest, well inside one node per 12 bytes) | program blobs
    // | proof tables, rebuilt levels and branches (pq)
    const size_t need = lit_cap + 32 * max_nodes + in_pad + 64ull * n + 32 * max_nodes + prog_bytes + 8192 +
                        (pq ? pq->dev_bytes : 0);
    uint8_t* arena = static_cast<uint8_t*>(dev_scratch(need));
    const size_t h_proofs = align_up(total, 256) + lit_cap + prog_bytes;   // after what plan_upload stages
    const size_t stage_bytes = h_proofs + (pq ? pq->host_bytes : 0) + 64ull * n + 1024;
    uint8_t* hst = static_cast<uint8_t*>(pinned_scratch(stage_bytes));
    if (!arena || !hst) return LHB200_ENOMEM;
    Plan pl;
    int32_t rc = build_plan(pl, arena, need, lit_cap, build, max_nodes);   // fails only on the node or literal cap
    if (bad) { set_error("BeaconBlock SSZ: malformed offsets or lengths for this fork"); return LHB200_EINVAL; }
    if (rc || pl.ops.size() + pl.items.size() > max_nodes || pl.bump + program_bytes(pl.ops.size(), pl.items.size()) > need) {
        set_error("internal: block plan exceeds its arena bound (%zu ops + %zu items of %zu nodes, %zu of %zu literal bytes, "
                  "%zu of %zu arena bytes)", pl.ops.size(), pl.items.size(), max_nodes, pl.lit.size(), lit_cap, pl.bump, need);
        return LHB200_ERETRY;
    }
    // the proofs are resolved over the finished plan; their tables and branches go after its program blobs
    std::unique_ptr<ProofResolver> pr;
    if (pq) {
        pr.reset(new ProofResolver(pl));
        for (uint32_t i = 0; i < pq->n; i++)
            if ((rc = pr->resolve(reinterpret_cast<uint64_t>(d_body + 32ull * pq->block_of[i]), pq->gindices[i]))) return rc;
        if (pr->table_bytes() > pq->host_bytes ||
            pl.bump + program_bytes(pl.ops.size(), pl.items.size()) + pr->device_bytes() > need) {
            set_error("internal: block proofs exceed their bound (%zu table bytes of %zu, %zu device bytes)",
                      pr->table_bytes(), pq->host_bytes, pr->device_bytes());
            return LHB200_EINVAL;
        }
    }
    memcpy(hst, ssz + base, total);
    memset(hst + total, 0, align_up(total, 256) - total);
    LHB_CUDA(cudaMemcpyAsync(d_in, hst, align_up(total, 256), cudaMemcpyHostToDevice, c.stream));
    rc = plan_upload(pl, c.stream, hst + align_up(total, 256));
    if (rc) return rc;
    if (pr && (rc = pr->upload(hst + h_proofs, pl.alloc(pr->device_bytes()), c.stream))) return rc;
    rc = plan_enqueue(pl, c.stream);
    if (rc) return rc;
    if (pr) {
        if ((rc = proof_events()) || (rc = pr->enqueue(c.stream, g_proof_ev[0], g_proof_ev[1]))) return rc;
        if (pr->first.back())
            LHB_CUDA(cudaMemcpyAsync(pq->branches, pr->d_branches, pr->first.back() * 32, cudaMemcpyDefault, c.stream));
    }
    uint8_t* h_out = hst + stage_bytes - 64ull * n - 64;
    LHB_CUDA(cudaMemcpyAsync(h_out, d_roots, 32ull * n, cudaMemcpyDeviceToHost, c.stream));
    if (body_roots) LHB_CUDA(cudaMemcpyAsync(h_out + 32ull * n, d_body, 32ull * n, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(roots, h_out, 32ull * n);
    if (body_roots) memcpy(body_roots, h_out + 32ull * n, 32ull * n);
    return LHB200_OK;
}

// n BeaconBlock SSZ blobs of `fork`, concatenated; offsets[n+1]; roots n*32; body_roots n*32 or NULL.
static int32_t block_roots(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, uint8_t* roots,
                                 uint8_t* body_roots, bool blinded, int32_t fork = LHB200_FORK_DENEB,
                                 BodyProofs* pq = nullptr) {
    LHB_REQUIRE_READY();
    const ForkLayout* fl = fork_layout(fork);
    if (!fl || (blinded && !fl->payload_fields)) {
        set_error("beacon_block_roots: fork id %d not supported (Altair .. Electra; blinded blocks from Bellatrix)", fork);
        return LHB200_EINVAL;
    }
    if (!ssz || !offsets || !roots || n == 0) { set_error("beacon_block_roots: null argument or zero blocks"); return LHB200_EINVAL; }
    for (uint32_t i = 0; i < n; i++)
        if (offsets[i] > offsets[i + 1]) { set_error("beacon_block_roots: offsets not monotone"); return LHB200_EINVAL; }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const uint64_t base = offsets[0], total = offsets[n] - offsets[0];
    const size_t in_pad = align_up(total + 64, 256);
    // Offset pre-scan: the only SSZ shape with more than one tree node per ~14 input bytes is a run of (near-)empty
    // transactions — a 4-byte offset each, one byte item + one list node + one length literal.  Count them per block
    // (a walk over its offsets) so the arena bound is tight for real blocks and still holds for that shape.
    uint64_t n_tx = 0;
    if (!blinded)
        for (uint32_t i = 0; i < n; i++) n_tx += prescan_transactions(ssz + offsets[i], offsets[i + 1] - offsets[i], *fl);
    if (pq) {   // bounds: one source per sibling, and one rebuilt tree per block (its DepositRequest list) of at most
                // one chunk per 192 input bytes, over at most 13 levels
        uint64_t siblings = 0;
        for (uint32_t i = 0; i < pq->n; i++) siblings += pq->gindices[i] ? 63 - __builtin_clzll(pq->gindices[i]) : 0;
        pq->host_bytes = align_up(pq->n * sizeof(ProofDesc), 256) + align_up((pq->n + 1) * 8ull, 256) +
                         align_up(siblings * sizeof(ProofSrc), 256) + 256 + align_up(n * sizeof(ProofTree), 256);
        pq->dev_bytes = pq->host_bytes + 32 * (total / 192) + n * 14 * 256ull + align_up(siblings * 32, 256) + 1024;
    }
    int32_t rc = LHB200_OK;
    for (int attempt = 0; attempt < 2; attempt++) {
        // attempt 0: transactions counted, everything else <= one node per 12 bytes and one literal per 8 bytes;
        // attempt 1 (only if a plan ever exceeds that): the unconditional bound of one node and literal per 2 bytes.
        const size_t max_nodes = attempt == 0 ? 2 * n_tx + total / 12 + 512ull * n : total / 2 + 512ull * n;
        const size_t lit_cap = align_up(32 * (attempt == 0 ? n_tx + total / 8 + 128ull * n : total / 2 + 128ull * n), 256);
        rc = block_roots_attempt(c, ssz, offsets, n, roots, body_roots, blinded, *fl, base, total, in_pad, max_nodes, lit_cap,
                                 pq);
        if (rc != LHB200_ERETRY) break;
    }
    return rc == LHB200_ERETRY ? LHB200_EINVAL : rc;
}
int32_t lhb200_beacon_block_roots_deneb(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, uint8_t* roots,
                                        uint8_t* body_roots) {
    return block_roots(ssz, offsets, n, roots, body_roots, false);
}
int32_t lhb200_beacon_block_root_deneb(const uint8_t* ssz, uint64_t len, uint8_t out[32], uint8_t* body_root) {
    const uint64_t offs[2] = {0, len};
    return block_roots(ssz, offs, 1, out, body_root, false);
}
// The variants of the BeaconBlock superstruct from Altair on (beacon_block.rs:41-90, beacon_block_body.rs:43-121): fork is
// LHB200_FORK_ALTAIR .. LHB200_FORK_ELECTRA; blinded != 0 selects the BlindedBeaconBlock form (Bellatrix and later).
int32_t lhb200_beacon_block_roots(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, int32_t fork, int32_t blinded,
                                  uint8_t* roots, uint8_t* body_roots) {
    return block_roots(ssz, offsets, n, roots, body_roots, blinded != 0, fork);
}
// Branches of generalized indices below the body roots of a block batch (BeaconBlockBody::kzg_commitment_merkle_proof,
// beacon_block_body.rs:178-227, and the other body proofs): one plan for the batch as lhb200_beacon_block_roots builds
// it, the proofs resolved over it before anything runs, and their branches gathered before the arena goes back.
int32_t lhb200_beacon_block_body_proofs(const uint8_t* ssz, const uint64_t* offsets, uint32_t n_blocks, int32_t fork,
                                        int32_t blinded, const uint32_t* block_of, const uint64_t* gindices, uint32_t n,
                                        uint8_t* branches, uint8_t* body_roots) {
    LHB_REQUIRE_READY();
    if (!body_roots || (n && (!block_of || !gindices))) { set_error("beacon_block_body_proofs: null argument"); return LHB200_EINVAL; }
    uint64_t siblings = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (block_of[i] >= n_blocks) {
            set_error("beacon_block_body_proofs: proof %u is taken in block %u of %u", i, block_of[i], n_blocks);
            return LHB200_EINVAL;
        }
        siblings += gindices[i] ? 63 - __builtin_clzll(gindices[i]) : 0;
    }
    if (siblings && !branches) { set_error("beacon_block_body_proofs: null branches"); return LHB200_EINVAL; }
    std::vector<uint8_t> roots(32ull * std::max<uint32_t>(n_blocks, 1));
    BodyProofs pq{block_of, gindices, n, branches, 0, 0};
    return block_roots(ssz, offsets, n_blocks, roots.data(), body_roots, blinded != 0, fork, &pq);
}
// BlindedBeaconBlock (beacon_block.rs:80): the body carries the ExecutionPayloadHeader; the root equals the full block's.
int32_t lhb200_blinded_beacon_block_roots_deneb(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, uint8_t* roots,
                                                uint8_t* body_roots) {
    return block_roots(ssz, offsets, n, roots, body_roots, true);
}

// swap_or_not_shuffle::shuffle_list(input, rounds, seed, forwards) (consensus/swap_or_not_shuffle/src/shuffle_list.rs:79).
// The reference returns None for an empty list, more than 2^24 elements or zero rounds: LHB200_EINVAL here.
int32_t lhb200_shuffle_list(const uint64_t* input, uint64_t n, uint8_t rounds, const uint8_t seed[32], int32_t forwards,
                            uint64_t* out) {
    LHB_REQUIRE_READY();
    if (!input || !out || !seed || n == 0 || n > (1ull << 24) || rounds == 0) {
        set_error("shuffle_list: empty list, more than 2^24 elements or zero rounds (reference returns None)");
        return LHB200_EINVAL;
    }
    Ctx& c = ctx();
    std::lock_guard<std::recursive_mutex> g(c.mu);
    const uint32_t n_blocks = (uint32_t)ceil_div(n, 256);
    const size_t b_in = align_up(n * 8, 256), b_src = align_up((size_t)rounds * n_blocks * 32, 256),
                 b_piv = 2048 + 256;   // 255 rounds x 8-byte pivots (2040 B), then the seed in its own slot
    uint8_t* d = static_cast<uint8_t*>(dev_scratch(2 * b_in + b_src + b_piv + 256));
    uint8_t* h = static_cast<uint8_t*>(pinned_scratch(2 * b_in + 64));
    if (!d || !h) return LHB200_ENOMEM;
    uint64_t* d_in = reinterpret_cast<uint64_t*>(d);
    uint64_t* d_out = reinterpret_cast<uint64_t*>(d + b_in);
    uint8_t* d_src = d + 2 * b_in;
    uint64_t* d_piv = reinterpret_cast<uint64_t*>(d_src + b_src);
    uint8_t* d_seed = reinterpret_cast<uint8_t*>(d_piv) + 2048;
    memcpy(h, input, n * 8);
    memcpy(h + b_in, seed, 32);
    LHB_CUDA(cudaMemcpyAsync(d_in, h, n * 8, cudaMemcpyHostToDevice, c.stream));
    LHB_CUDA(cudaMemcpyAsync(d_seed, h + b_in, 32, cudaMemcpyHostToDevice, c.stream));
    const uint64_t total = std::max<uint64_t>((uint64_t)rounds * n_blocks, rounds);
    k_shuffle_hashes<<<(unsigned)ceil_div(total, 128), 128, 0, c.stream>>>(d_seed, rounds, n, n_blocks, d_piv, d_src);
    k_shuffle_permute<<<(unsigned)ceil_div(n, 256), 256, 0, c.stream>>>(d_in, d_out, n, rounds, n_blocks, d_piv, d_src,
                                                                        forwards ? 1 : 0);
    count_launch(2);
    LHB_CUDA(cudaGetLastError());
    LHB_CUDA(cudaMemcpyAsync(h, d_out, n * 8, cudaMemcpyDeviceToHost, c.stream));
    LHB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out, h, n * 8);
    return LHB200_OK;
}

}  // extern "C"
