/*
 * lhb200.h — C ABI of liblhb200.so: the H100-native (sm_90a) replacement for Lighthouse's two
 * compute-bound hot paths.  Plain pointers and sizes only; no exceptions or panics cross this boundary.
 *
 * Citations are file:line under sigp/lighthouse v5.3.0 (/root/reference).  The Rust-side bindings a
 * Lighthouse maintainer would add are shown in INTEGRATION.md.
 *
 * Conventions
 *   - Every entry point returns an int32 status: LHB200_OK (0) or a negative LHB200_E* code;
 *     lhb200_last_error() gives a thread-local human-readable message.  Results go to out-params.
 *   - "Host" entry points take caller-owned host buffers that are only read during the call (they mirror
 *     the borrowed Cow<'a, ..> data of bls::SignatureSet / &self of TreeHash); nothing is retained.
 *   - "dev_" entry points take device pointers (inputs already resident in HBM) and an optional
 *     cudaStream_t passed as void* (NULL = the library's stream); they return after enqueueing unless
 *     documented otherwise.
 *   - There is NO CPU fallback: without a usable sm_90 device every compute entry point returns
 *     LHB200_ENODEV.
 */
#ifndef LHB200_H
#define LHB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LHB200_API __attribute__((visibility("default")))
#else
#define LHB200_API
#endif

#define LHB200_OK 0
#define LHB200_ENODEV (-1)   /* no CUDA device / init not called / init failed */
#define LHB200_EINVAL (-2)   /* bad argument (null pointer, inconsistent sizes, malformed SSZ offsets) */
#define LHB200_ECUDA (-3)    /* CUDA runtime error (message in lhb200_last_error) */
#define LHB200_ENOMEM (-4)   /* device or pinned allocation failed */
#define LHB200_EDECODE (-5)  /* a serialized point failed to decode (bls::Error::InvalidByteLength/BlstError) */

/* ---- lifecycle -------------------------------------------------------------------------------- */

/* Bind the calling process to CUDA device `device` (one process per GPU), create the library stream and
 * scratch arenas and upload constant tables.  Idempotent for the same device. */
LHB200_API int32_t lhb200_init(int32_t device);
LHB200_API void lhb200_shutdown(void);
LHB200_API const char* lhb200_last_error(void);
/* Pinned host memory for callers that want zero-staging H2D (the e2e bench uses it). */
LHB200_API int32_t lhb200_pinned_alloc(void** out, uint64_t nbytes);
LHB200_API int32_t lhb200_pinned_free(void* p);
/* Number of kernel launches issued by this library since init (bench.py's "gpu_launches"). */
LHB200_API uint64_t lhb200_launch_count(void);

/* ---- tree-hash path --------------------------------------------------------------------------- */

/* ethereum_hashing::hash32_concat over n independent 64-byte inputs (consensus/merkle_proof/src/lib.rs:91,
 * :380-384): out[i] = SHA256(in[64i .. 64i+64]). */
LHB200_API int32_t lhb200_hash_pairs(const uint8_t* in, uint8_t* out, uint64_t n);
LHB200_API int32_t lhb200_dev_hash_pairs(const void* d_in, void* d_out, uint64_t n, void* stream);

/* tree_hash::merkle_root / merkleize with a chunk limit of 2^depth (crypto/bls/src/macros.rs:24,
 * SURVEY Appendix B): zero-pads every level with ZERO_HASHES[level]; n_chunks == 0 gives ZERO_HASHES[depth].
 * n_chunks must be <= 2^depth. */
LHB200_API int32_t lhb200_merkleize(const uint8_t* chunks, uint64_t n_chunks, uint32_t depth, uint8_t out[32]);
/* d_chunks must be 16-byte aligned; d_out32 receives the 32-byte root (device memory). */
LHB200_API int32_t lhb200_dev_merkleize(const void* d_chunks, uint64_t n_chunks, uint32_t depth, void* d_out32, void* stream);

/* tree_hash::mix_in_length(root, len) = SHA256(root || le64(len) || 0^24). */
LHB200_API int32_t lhb200_mix_in_length(const uint8_t root[32], uint64_t len, uint8_t out[32]);

/* ZERO_HASHES[depth] (ethereum_hashing::ZERO_HASHES, merkle_proof/src/lib.rs:166), depth <= 64. */
LHB200_API int32_t lhb200_zero_hash(uint32_t depth, uint8_t out[32]);

/* hash_tree_root(List[Validator, 2^40]) from n 121-byte SSZ validators (consensus/types/src/validator.rs:25-35;
 * beacon_state.rs:363).  lhb200_validator_roots writes the n per-validator roots instead. */
LHB200_API int32_t lhb200_validators_root(const uint8_t* ssz, uint64_t n, uint8_t out[32]);
LHB200_API int32_t lhb200_validator_roots(const uint8_t* ssz, uint64_t n, uint8_t* out_roots);

/* BeaconState::update_tree_hash_cache / tree_hash_root for the Deneb variant, mainnet preset, cold (no cached
 * nodes) — consensus/types/src/beacon_state.rs:2031-2038, fields :343-484.  `ssz` is the SSZ encoding of
 * BeaconStateDeneb.  field_roots (28*32 bytes) is optional (NULL to skip). */
LHB200_API int32_t lhb200_beacon_state_root_deneb(const uint8_t* ssz, uint64_t len, uint8_t out[32], uint8_t* field_roots);
/* The other variants of the BeaconState superstruct (consensus/types/src/beacon_state.rs:224-571) through the same
 * kernels; `fork` is one of LHB200_FORK_*.  Base (phase0) has 21 fields, whose 15 and 16 are previous_ /
 * current_epoch_attestations: List[PendingAttestation, 4096] (pending_attestation.rs:25-32), rooted by one
 * k_pending_attestation_roots launch for both lists.  Altair has 24 fields, Bellatrix 25 (+ a 14-field execution
 * payload header), Capella 28 (15-field header, withdrawal indices, historical_summaries), Deneb 28 (17-field header).
 * field_roots (optional, 28 x 32 B): entries beyond the fork's field count are zero chunks. */
#define LHB200_FORK_BASE 0
#define LHB200_FORK_ALTAIR 1
#define LHB200_FORK_BELLATRIX 2
#define LHB200_FORK_CAPELLA 3
#define LHB200_FORK_DENEB 4
#define LHB200_FORK_ELECTRA 5   /* 37 fields (19-field header, six u64s, three pending_* lists): field_roots is 37 x 32 B */
LHB200_API int32_t lhb200_beacon_state_root(const uint8_t* ssz, uint64_t len, int32_t fork, uint8_t out[32],
                                            uint8_t* field_roots);
LHB200_API int32_t lhb200_state_stage(const uint8_t* ssz, uint64_t len, int32_t fork, struct lhb200_state** out);

/* Device-resident variant: stage once (H2D into the library's aligned HBM layout, DESIGN.md §3), then hash
 * as often as wanted without touching the host link.  The handle owns device memory until released. */
typedef struct lhb200_state lhb200_state;
LHB200_API int32_t lhb200_state_stage_deneb(const uint8_t* ssz, uint64_t len, lhb200_state** out);
LHB200_API int32_t lhb200_state_root(lhb200_state* st, uint8_t out[32], uint8_t* field_roots);
/* Same-length in-place mutation of a staged state — the resident analogue of apply_pending_mutations
 * (beacon_state.rs:2459-2481): bytes [ssz_offset, ssz_offset+len) of the SSZ encoding are replaced; the next
 * lhb200_state_root re-hashes everything on the device (SURVEY.md §8f-3: warm path = patch + full re-hash).  On a Base
 * handle a range inside previous_ / current_epoch_attestations gives LHB200_EINVAL (and the batch changes nothing):
 * those lists change through lhb200_state_set_pending_attestations, which checks them. */
LHB200_API int32_t lhb200_state_patch(lhb200_state* st, uint64_t ssz_offset, const uint8_t* data, uint64_t len);
/* n non-overlapping same-length mutations in one call (offsets[i], lens[i], bytes concatenated in `data`): one H2D copy
 * and one scatter kernel instead of n round trips — what a slot's worth of milhouse pending updates looks like. */
LHB200_API int32_t lhb200_state_patch_batch(lhb200_state* st, const uint64_t* offsets, const uint32_t* lens,
                                            const uint8_t* data, uint32_t n);
/* Warm path (SURVEY.md §8f-3; the reference's steady state: BeaconState::update_tree_hash_cache re-hashes only dirty
 * paths, beacon_state.rs:2031-2038,2459-2481).  After this call the handle keeps every level of its big lists
 * (validators, balances, inactivity scores, participation x2, randao mixes, block/state roots, slashings) resident:
 * lhb200_state_patch marks the leaves it touches and lhb200_state_root / _enqueue re-hash only the paths above them
 * plus the tail program.  The first root after enabling is cold (it builds the levels); patches to other lists, or
 * more than 65 536 dirty leaves, fall back to a cold root.  Unsharded handles only.  With lhb200_state_root_enqueue the
 * dirty-leaf table is staged through the library's pinned slab: synchronise the stream before the next lhb200_* call
 * (lhb200_state_root does).
 * lhb200_state_last_root_hashes: hash32_concat units the last root actually computed. */
LHB200_API int32_t lhb200_state_enable_incremental(lhb200_state* st);
LHB200_API uint64_t lhb200_state_last_root_hashes(const lhb200_state* st);
/* Resizable lists of an incremental, unsharded handle: what a block and an epoch do to list lengths (eth1 votes,
 * deposits, historical_summaries, Electra's pending lists) without re-staging.  One edit per field and call:
 *   append     first = old_len, new_len = old_len + n        truncate / reset   n = 0, new_len < old_len
 *   front drain  first = 0, n = new_len (the remaining items)  rewrite            new_len = old_len
 * Items [first, first + n) are written from `data` (SSZ bytes, edit after edit); first + n <= new_len and every item
 * in [old_len, new_len) must be written.  Fields (container index, item bytes): 9 eth1_data_votes (72), 11 validators
 * (121), 12 balances (8), 15 / 16 previous_ / current_epoch_participation (1), 21 inactivity_scores (8),
 * 27 historical_summaries (64, Capella and later), 34 / 35 / 36 pending_balance_deposits / pending_partial_withdrawals /
 * pending_consolidations (16 / 24 / 16, Electra).  Base has 9, 11 and 12 only (see
 * lhb200_state_set_pending_attestations for its fields 15 and 16).  historical_roots is not resizable.  A field the fork does not have,
 * a limit overrun, reserved != 0, or a non-incremental or sharded handle gives LHB200_EINVAL, and a refused call
 * changes nothing.  Afterwards roots, field roots, hash units and lhb200_state_patch offsets all refer to the current
 * encoding; bytes past a list's length are not resident.  Only the dirty paths, the changed lists' zero ladders and
 * length mix-ins and the tail program are re-hashed; more than 65 536 dirty leaves in one list re-hash its tree from
 * the resident items. */
typedef struct lhb200_list_edit {
    uint32_t field;     /* index in the state container (field_roots order) */
    uint32_t reserved;  /* 0 */
    uint64_t new_len;   /* item count after the edit */
    uint64_t first;     /* first item written */
    uint64_t n;         /* items written; their SSZ bytes follow in `data`, edit after edit */
} lhb200_list_edit;
LHB200_API int32_t lhb200_state_list_edit(lhb200_state* st, const lhb200_list_edit* edits, uint32_t n_edits,
                                          const uint8_t* data);
/* Current item count of resizable list `field` (see lhb200_state_list_edit). */
LHB200_API int32_t lhb200_state_list_len(const lhb200_state* st, uint32_t field, uint64_t* len);
/* Replace latest_execution_payload_header (Bellatrix and later) with `len` bytes of SSZ of the handle's fork; its
 * extra_data may change length.  Same handle requirements as lhb200_state_list_edit. */
LHB200_API int32_t lhb200_state_set_payload_header(lhb200_state* st, const uint8_t* ssz, uint64_t len);
/* Base: replace previous_epoch_attestations (field 15) or current_epoch_attestations (16) with `len` bytes of SSZ of a
 * List[PendingAttestation, 4096] — per block the current list plus the block's attestations, at the epoch boundary
 * two calls (current -> previous, then an empty current).  Same handle requirements as lhb200_state_list_edit, whose
 * storage holds 4096 records of the largest size.  Another fork or field, malformed SSZ (offset table, record sizes,
 * bitlist delimiter, more than 2048 bits or 4096 records) -> LHB200_EINVAL, and a refused call changes nothing.
 * Afterwards lhb200_state_patch offsets and lhb200_state_list_len (which gives the record count of 15 / 16 on a Base
 * handle) refer to the new encoding.  The next root re-roots every record of both lists (one launch,
 * ~19 hashes a record) and re-hashes the replaced list's tree above the slots that changed. */
LHB200_API int32_t lhb200_state_set_pending_attestations(lhb200_state* st, uint32_t field, const uint8_t* ssz,
                                                         uint64_t len);
/* Same as lhb200_state_root but only enqueues; the root lands in device memory (returned pointer valid until
 * the next call on this handle).  Used by bench.py to time kernels with CUDA events. */
LHB200_API int32_t lhb200_state_root_enqueue(lhb200_state* st, void* stream, const void** d_root);
/* One state sharded over `world` GPUs (a power of two; SURVEY.md §8e): rank r stages and hashes only its leaf range
 * of the big lists (validators, balances, randao_mixes, participation x2, inactivity_scores) plus the small fields.
 *   1. lhb200_state_stage_deneb_shard(ssz, len, rank, world, &h)       every rank, its own slice
 *   2. lhb200_state_shard_roots(h, roots, &n)                          n x 32-byte subtree roots of this rank
 *   3. all-gather the n*32 bytes over NCCL (rank-major)                 the path's single collective
 *   4. lhb200_state_combine(h, gathered, out)                          every rank: log2(world) levels + ladders + top tree */
LHB200_API int32_t lhb200_state_stage_deneb_shard(const uint8_t* ssz, uint64_t len, uint32_t rank, uint32_t world,
                                                  lhb200_state** out);
LHB200_API int32_t lhb200_state_shard_roots(lhb200_state* st, uint8_t* out, uint32_t* n_lists);
LHB200_API int32_t lhb200_state_combine(lhb200_state* st, const uint8_t* gathered, uint8_t out[32]);
/* Steps 2-4 in one call over the library's communicator (lhb200_comm_init): subtree roots stay on the device, one
 * ncclAllGather, every rank folds the top; only the 32-byte root crosses the host link. */
LHB200_API int32_t lhb200_state_root_sharded(lhb200_state* st, uint8_t out[32]);
LHB200_API int32_t lhb200_state_release(lhb200_state* st);
/* BeaconState::clone of a resident, unsharded handle: a new handle with the same fork, encoding, list lengths and
 * capacities, payload header, incremental / converted status and pending (not yet rooted) mutations, whose device
 * memory is its own.  Afterwards the two are independent: edits, roots and release of one never affect the other.
 * Blocks until the clone is ready; work enqueued on `src` through lhb200_state_root_enqueue on another stream must be
 * complete.  The live bytes are copied by one kernel launch.  Sharded handle -> LHB200_EINVAL; on failure *out is
 * untouched and src unchanged. */
LHB200_API int32_t lhb200_state_clone(const lhb200_state* src, lhb200_state** out);
/* HBM held by the handle (arena, levels, tree and dirty tables, resizable-list storage), for cache sizing. */
LHB200_API int32_t lhb200_state_device_bytes(const lhb200_state* st, uint64_t* bytes);
/* Test hook: *disjoint = 1 iff no device address held by `a` lies in an allocation of `b`. */
LHB200_API int32_t lhb200_debug_state_disjoint(const lhb200_state* a, const lhb200_state* b, int32_t* disjoint);
/* Test hook: the live bytes lhb200_state_clone copies for this handle (its arena up to the allocation cursor, its
 * levels, and each resizable list up to its length). */
LHB200_API int32_t lhb200_debug_state_live_bytes(const lhb200_state* st, uint64_t* bytes);
/* Algorithmic work of the last root computed on this handle: number of hash32_concat units. */
LHB200_API uint64_t lhb200_state_hash_units(const lhb200_state* st);
/* Device time (ms) of the dominant kernel (k_validator_roots) in the last completed root, from CUDA events on the
 * launching stream; < 0 if unavailable. */
LHB200_API float lhb200_state_dominant_kernel_ms(const lhb200_state* st);

/* MerkleTree::create(leaves, depth) + generate_proof(index, depth) (consensus/merkle_proof/src/lib.rs:68-99,
 * :290-324): root and the bottom-up branch (depth * 32 bytes).  n <= 2^depth, depth <= 32. */
LHB200_API int32_t lhb200_merkle_tree_proof(const uint8_t* leaves, uint64_t n, uint32_t depth, uint64_t index, uint8_t root[32],
                                 uint8_t* branch);
/* verify_merkle_proof / merkle_root_from_branch batch (merkle_proof/src/lib.rs:357-389): for each i,
 * ok[i] = (fold(leaf_i, branch_i, depth, index_i) == root_i).  branches: n * depth * 32 bytes. */
LHB200_API int32_t lhb200_verify_merkle_proofs(const uint8_t* leaves, const uint8_t* branches, uint32_t depth,
                                    const uint64_t* indices, const uint8_t* roots, uint64_t n, uint8_t* ok);
/* Branches of generalized indices of a resident BeaconState (spec compute_merkle_proof, consensus-specs
 * ssz/merkle-proofs.md; beacon_state.rs:2483).  Roots the handle first, warm or cold exactly as lhb200_state_root
 * would, consuming pending mutations the same way.  Proof i has depth_i = floor(log2(gindices[i])) siblings, bottom-up
 * (the leaf's sibling first), at branches + 32 * sum_{j<i} depth_j.  root: the state root every branch verifies
 * against.  Unsharded handles of every fork, incremental or not, converted or not.  LHB200_EINVAL, with the handle
 * left as it was: gindex 0, a gindex below a leaf (a u64 field, a packed chunk, a validator, record or byte-string
 * root), a sharded handle.  One gather launch per call, plus one k_tree_level launch per level the call rebuilds for a
 * list without resident levels. */
LHB200_API int32_t lhb200_state_proofs(lhb200_state* st, const uint64_t* gindices, uint32_t n, uint8_t* branches,
                                       uint8_t root[32]);
/* Same for the BeaconBlockBody of n_blocks blocks (SSZ and layout of lhb200_beacon_block_roots): gindices relative to
 * the BODY root, proof i taken in block block_of[i]; body_roots n_blocks x 32.  block_of[i] >= n_blocks, malformed
 * SSZ or a gindex below a leaf (a transaction, a signature, a commitment root) -> LHB200_EINVAL. */
LHB200_API int32_t lhb200_beacon_block_body_proofs(const uint8_t* ssz, const uint64_t* offsets, uint32_t n_blocks,
                                                   int32_t fork, int32_t blinded, const uint32_t* block_of,
                                                   const uint64_t* gindices, uint32_t n, uint8_t* branches,
                                                   uint8_t* body_roots);
/* Benchmark hook: device time (ms) of the last k_proof_branches launch of either call above, from CUDA events recorded
 * around it; < 0 if unavailable. */
LHB200_API float lhb200_debug_proof_gather_ms(void);

/* BeaconBlock::canonical_root for BeaconBlockDeneb SSZ bytes, mainnet preset (consensus/types/src/beacon_block.rs:
 * 56-78,158-160; body beacon_block_body.rs:70-121,145-176; payload execution_payload.rs:54-95; operations
 * proposer_slashing.rs:26, attester_slashing.rs:42, indexed_attestation.rs:53, attestation.rs:74, deposit.rs:27,
 * signed_voluntary_exit.rs:25, sync_aggregate.rs:38, signed_bls_to_execution_change.rs:22, withdrawal.rs:22).
 * `body_root` (32 B, optional) receives hash_tree_root(body) — the BeaconBlockHeader.body_root of the block.
 * The batch form hashes n blocks (SSZ blobs concatenated, offsets[n+1]) in one pass: the 32 blocks of an epoch
 * segment (BlockSignatureVerifier / ConsensusContext::get_current_block_root, consensus_context.rs:115-128).
 * Malformed SSZ (bad offsets, over-limit lists, missing bitlist delimiter) -> LHB200_EINVAL. */
LHB200_API int32_t lhb200_beacon_block_root_deneb(const uint8_t* ssz, uint64_t len, uint8_t out[32], uint8_t* body_root);
LHB200_API int32_t lhb200_beacon_block_roots_deneb(const uint8_t* ssz, const uint64_t* offsets, uint32_t n,
                                                   uint8_t* roots, uint8_t* body_roots);
/* Same for BlindedBeaconBlockDeneb SSZ (BlindedBeaconBlock, consensus/types/src/beacon_block.rs:80; the body carries
 * the ExecutionPayloadHeaderDeneb, execution_payload_header.rs:46-87).  The root equals the full block's root. */
LHB200_API int32_t lhb200_blinded_beacon_block_roots_deneb(const uint8_t* ssz, const uint64_t* offsets, uint32_t n,
                                                           uint8_t* roots, uint8_t* body_roots);
/* The same for every variant of the BeaconBlock superstruct from Base on (consensus/types/src/beacon_block.rs:19-90,
 * beacon_block_body.rs:33-121): fork = LHB200_FORK_BASE (8 body fields: Altair's without sync_aggregate),
 * _ALTAIR (9 body fields, no execution payload), _BELLATRIX (14-field
 * payload), _CAPELLA (+ withdrawals, bls_to_execution_changes), _DENEB (+ blob gas fields, blob_kzg_commitments),
 * _ELECTRA (+ consolidations; attestations with committee_bits and up to 131 072 aggregation bits, at most 8 of them
 * and 1 attester slashing; payload + deposit_requests (<= 8192) and withdrawal_requests (<= 16),
 * execution_payload.rs:54-101, attestation.rs:76-82, deposit_request.rs:23-29, signed_consolidation.rs:23-24);
 * blinded != 0: BlindedBeaconBlock (the body carries the ExecutionPayloadHeader; Bellatrix and later). */
LHB200_API int32_t lhb200_beacon_block_roots(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, int32_t fork,
                                             int32_t blinded, uint8_t* roots, uint8_t* body_roots);

/* swap_or_not_shuffle::shuffle_list (consensus/swap_or_not_shuffle/src/shuffle_list.rs:79-160; SURVEY.md §8f-4):
 * out = shuffle (forwards != 0) or un-shuffle (forwards == 0, the direction the spec uses for committees) of the n
 * 64-bit values of `input`.  n == 0, n > 2^24 or rounds == 0 -> LHB200_EINVAL (the reference returns None). */
LHB200_API int32_t lhb200_shuffle_list(const uint64_t* input, uint64_t n, uint8_t rounds, const uint8_t seed[32],
                                       int32_t forwards, uint64_t* out);

/* Committees, proposers and the next sync committee of a resident, unsharded BeaconState of any fork (mainnet preset,
 * reference semantics for every fork from Base to Electra).  They read the handle's validator records, randao_mixes
 * and slot on the device, as patches, list edits and clones left them, and change nothing a later root, clone or
 * proof sees.  Refusals -> LHB200_EINVAL with lhb200_last_error set: a sharded handle, a cap below the validator
 * count, an epoch out of bounds (checked before anything is launched); no validator active at the epoch, or more
 * than 2^24 active (found by the counting pass, which writes only library scratch).  Each call makes a fixed number
 * of launches and one synchronise before its final copy. */
typedef struct {
    uint64_t epoch, n_validators, n_active, committees_per_slot;
    uint8_t seed[32];                       /* get_seed(epoch, DOMAIN_BEACON_ATTESTER) */
} lhb200_committee_info;
/* CommitteeCache::initialized(state, epoch) (committee_cache.rs:64-125): shuffling[0..n_active) = shuffle_list(active
 * indices, 90, seed, forwards = false); positions[0..n_validators) (0 = None, else position + 1; may be NULL).  cap =
 * entries each buffer holds, at least the handle's validator count.  The epoch is out of bounds when epoch - 2 (saturating)
 * is below min_randao_epoch = current_epoch + 1 - 65536 (saturating), or when it is above current_epoch + 1. */
LHB200_API int32_t lhb200_state_committee_cache(lhb200_state* st, uint64_t epoch, uint64_t* shuffling,
                                               uint32_t* positions, uint64_t cap, lhb200_committee_info* info);
/* get_beacon_proposer_indices (beacon_state.rs:1025-1037): the proposer of each slot of the current epoch. */
LHB200_API int32_t lhb200_state_beacon_proposer_indices(lhb200_state* st, uint64_t out[32]);
/* get_next_sync_committee_indices (beacon_state.rs:1091-1125): 512 indices drawn at current_epoch + 1, duplicates
 * kept. */
LHB200_API int32_t lhb200_state_next_sync_committee_indices(lhb200_state* st, uint64_t out[512]);
/* A committee cache that stays on the device: the same steps, refusals and messages as lhb200_state_committee_cache
 * (5 launches, the one read-back of the active count), with the shuffling left in device memory the handle owns.  The handle does not depend
 * on the state once created: releasing, patching or cloning the state leaves it as it is (Lighthouse keeps committee
 * caches across states).  lhb200_committee_cache_shuffling copies the n_active shuffled indices out (one copy; cap =
 * entries `out` holds, at least info.n_active).  Release frees the handle (NULL is a no-op). */
typedef struct lhb200_committee_cache lhb200_committee_cache;
LHB200_API int32_t lhb200_state_committee_cache_create(lhb200_state* st, uint64_t epoch, lhb200_committee_cache** out);
LHB200_API int32_t lhb200_committee_cache_info(const lhb200_committee_cache* cc, lhb200_committee_info* info);
LHB200_API int32_t lhb200_committee_cache_shuffling(const lhb200_committee_cache* cc, uint64_t* out, uint64_t cap);
LHB200_API int32_t lhb200_committee_cache_release(lhb200_committee_cache* cc);

/* ---- BLS batch verification path ---------------------------------------------------------------- */

/* bls::verify_signature_sets (crypto/bls/src/impls/blst.rs:37-119) over SoA-flattened SignatureSets
 * (crypto/bls/src/generic_signature_set.rs:61-121):
 *   sigs        n x 96 B  compressed G2 (ZCash format; all-zero = Lighthouse's "empty" signature -> false)
 *   msgs        n x 32 B  signing roots
 *   pks         K x 96 B  uncompressed affine G1, x || y big-endian (the validator_pubkey_cache.rs:195-199 format;
 *                         keys are NOT re-validated, matching pks_validate=false at blst.rs:115).  Keys must be in
 *                         G1: sets that share a message are paired once, through the sum of their r_i apk_i, and
 *                         prod_i e(r_i apk_i, H(m)) = e(sum_i r_i apk_i, H(m)) rests on bilinearity, which holds for
 *                         G1 points.  Lighthouse's keys are (validated at import, validator_pubkey_cache.rs:116-118).
 *   pk_offsets  n+1 u32   CSR: set i owns keys [pk_offsets[i], pk_offsets[i+1])
 *   rands       n x u64   nonzero random scalars (blst.rs:55-67), or NULL to have the library draw them
 * *ok = 1 iff  prod_i e(r_i apk_i, H(m_i)) == e(g1, sum_i r_i sig_i)  and every set passed its checks
 * (non-empty, subgroup-checked signature; >= 1 key; aggregate key not at infinity).  n_sets == 0 -> *ok = 0
 * (blst.rs:42-44).  set_status (optional, n bytes): 0 fine, 1 empty sig, 2 sig decode, 3 sig not in subgroup,
 * 4 no keys, 5 aggregate key at infinity, 6 key decode.  A set that fails several checks reports one code, in the
 * order blst.rs:73-106 checks them: a signature failure (1, 2, 3) first, then no keys (4), then key decode (6), then
 * the aggregate key at infinity (5).  fast_aggregate_verify / Signature::verify (blst.rs:196-200, :250-261) are the
 * n_sets == 1 case.
 * Sets that share a message (every unaggregated attestation of a committee, every sync-committee message of a slot)
 * are grouped: when at least one set in eight repeats a message, hash-to-G2 and the Miller loop run once per distinct
 * message over the sum of the group's r_i apk_i.  The verdict, the statuses and the final-exponentiated product are the same as without.
 * Concurrent calls of at most 64 sets are coalesced: a call that finds a free slot (at most sixteen passes run at
 * once) runs alone, as above.  A call that arrives while every slot is taken validates its arguments in its own thread
 * (an argument error is returned to that caller alone, as above), draws its own scalars when rands is NULL, and waits.
 * When a slot frees, the first waiting call takes the waiting calls that fit one segmented pass (see
 * lhb200_verify_signature_set_batches) and verifies them in one device pass, each as its own batch with its own
 * scalars, so its verdict and statuses are the ones it would get alone.  A CUDA error (or an allocation failure) in a
 * shared pass is returned to every call of that pass.  The call blocks until its own result is written. */
LHB200_API int32_t lhb200_verify_signature_sets(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                                const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets,
                                                uint8_t* ok, uint8_t* set_status);
/* n_batches independent verify_signature_sets calls in one: batch k is sets [batch_offsets[k], batch_offsets[k + 1])
 * of the SoA buffers above (pk_offsets over all n_sets sets), and ok[k] is exactly what lhb200_verify_signature_sets
 * gives for batch k alone with the same scalars; an empty batch gives 0 (blst.rs:42-44).  set_status (optional,
 * n_sets bytes) as above.  Consecutive batches are packed into segmented passes: one device pass runs the per-set
 * stages over all of a pass's sets, then per batch one sum of r_i sig_i, one pair (-g1, sum) and one final
 * exponentiation, so no batch's verdict depends on another's sets.  A pass holds batches while their sets plus their
 * count stay within 8 x the SM count (the warps of one wave of the one-warp-per-pairing Miller kernel); a batch too
 * large for a pass alone runs through lhb200_verify_signature_sets.  n_batches == 0 does nothing.  Non-monotone or
 * inconsistent offsets, a zero scalar or a null pointer -> LHB200_EINVAL ("verify_signature_set_batches: <reason>"). */
LHB200_API int32_t lhb200_verify_signature_set_batches(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                                       const uint32_t* pk_offsets, const uint64_t* rands,
                                                       uint32_t n_sets, const uint32_t* batch_offsets,
                                                       uint32_t n_batches, uint8_t* ok, uint8_t* set_status);

/* Staged form of the same call (what bench.py times): create once, upload or point at device-resident inputs,
 * enqueue on a stream, read the verdict.  The three host uploads (lhb200_bls_batch_upload, _upload_async,
 * _upload_indexed) group the sets by message on the host when at least one set in eight repeats a message, and
 * verify_enqueue then runs
 * hash-to-G2, the Miller loop and the product tree over the distinct messages (kernels and launch shapes chosen for
 * that count) after one per-message sum of the key stage's points.  Other batches, and inputs bound with
 * lhb200_bls_batch_set_device_inputs, run per set.  LHB_GROUP_MESSAGES=0 turns the grouping off. */
typedef struct lhb200_bls_batch lhb200_bls_batch;
LHB200_API int32_t lhb200_bls_batch_create(uint32_t max_sets, uint64_t max_keys, lhb200_bls_batch** out);
LHB200_API int32_t lhb200_bls_batch_destroy(lhb200_bls_batch* b);
LHB200_API int32_t lhb200_bls_batch_upload(lhb200_bls_batch* b, const uint8_t* sigs, const uint8_t* msgs,
                                           const uint8_t* pks, const uint32_t* pk_offsets, const uint64_t* rands,
                                           uint32_t n_sets);
LHB200_API int32_t lhb200_bls_batch_set_device_inputs(lhb200_bls_batch* b, const void* d_sigs, const void* d_msgs,
                                                      const void* d_pks, const void* d_offsets, const void* d_rands,
                                                      uint32_t n_sets);
/* Streamed upload: queues the small arrays on `stream` and binds the host key buffer; the host buffers must stay valid
 * and unchanged until lhb200_bls_batch_result returns.  verify_enqueue copies the keys in chunks of whole sets on
 * high-priority streams and aggregates each chunk as it lands while the signature and hash-to-curve kernels already run,
 * so the 1.2 GB of keys of a 100 k x 128 batch cross the host link behind the ALU-bound kernels (SURVEY.md §8d (ii):
 * "H2D must be double-buffered against compute").  lhb200_verify_signature_sets uses this path. */
LHB200_API int32_t lhb200_bls_batch_upload_async(lhb200_bls_batch* b, const uint8_t* sigs, const uint8_t* msgs,
                                                 const uint8_t* pks, const uint32_t* pk_offsets, const uint64_t* rands,
                                                 uint32_t n_sets, void* stream);
LHB200_API int32_t lhb200_bls_batch_verify_enqueue(lhb200_bls_batch* b, void* stream);
LHB200_API int32_t lhb200_bls_batch_result(lhb200_bls_batch* b, void* stream, uint8_t* ok, uint8_t* set_status);
/* Segmented pass, staged form (lhb200_verify_signature_set_batches splits its input into such passes): the sets of
 * the next upload are n_batches independent batches, batch k = sets [batch_offsets[k], batch_offsets[k + 1]).  Call
 * before the upload (the upload groups messages within each batch only; any earlier upload on `b` is dropped); the
 * next verify_enqueue checks every batch on its own and consumes the segments.  Batches must be non-empty, offsets
 * start at 0 and increase, and sets + n_batches must fit one pass (8 x the SM count) -> else LHB200_EINVAL.  The
 * upload must then carry batch_offsets[n_batches] sets.
 * lhb200_bls_batch_segment_result: ok[k] per batch (n_batches bytes) and, optionally, the per-set statuses.
 * lhb200_bls_batch_segment_gt: test hook, batch k's final-exponentiated product in the format of lhb200_bls_batch_gt
 * (zeros for a batch with a failed set). */
LHB200_API int32_t lhb200_bls_batch_set_segments(lhb200_bls_batch* b, const uint32_t* batch_offsets, uint32_t n_batches);
LHB200_API int32_t lhb200_bls_batch_segment_result(lhb200_bls_batch* b, void* stream, uint8_t* ok, uint8_t* set_status);
LHB200_API int32_t lhb200_bls_batch_segment_gt(lhb200_bls_batch* b, uint32_t k, uint8_t out576[576]);
/* Device-resident validator pubkey table — the mirror of ValidatorPubkeyCache
 * (beacon_node/beacon_chain/src/validator_pubkey_cache.rs:20-25,138-140; same 96-byte key format it persists, :195-199).
 * Keys are decoded to Montgomery form once at import; SignatureSets then carry u32 validator indices
 * (what consensus/state_processing/src/per_block_processing/signature_sets.rs:315-320 gathers) instead of 96-byte keys:
 * 512 B instead of 12 288 B per 128-key set on the host link (SURVEY.md §8f-1). */
typedef struct lhb200_pubkey_table lhb200_pubkey_table;
LHB200_API int32_t lhb200_pubkey_table_create(uint64_t capacity, lhb200_pubkey_table** out);
LHB200_API int32_t lhb200_pubkey_table_destroy(lhb200_pubkey_table* t);
LHB200_API int32_t lhb200_pubkey_table_append(lhb200_pubkey_table* t, const uint8_t* pks96, uint64_t n);
LHB200_API uint64_t lhb200_pubkey_table_len(const lhb200_pubkey_table* t);
LHB200_API int32_t lhb200_bls_batch_upload_indexed(lhb200_bls_batch* b, const lhb200_pubkey_table* table,
                                                   const uint8_t* sigs, const uint8_t* msgs, const uint32_t* key_indices,
                                                   const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets);
/* Attestations verified against resident committee caches and the pubkey table: get_attesting_indices
 * (get_attesting_indices.rs), indexed_attestation_signature_set (signature_sets.rs:271-332) and verify_signature_sets,
 * with the committee lookup, attesting indices, AttestationData and signing roots and the key gather on the device.
 *   ssz, offsets  n Attestation encodings, record i = ssz[offsets[i] .. offsets[i + 1]).  fork = LHB200_FORK_*: Base
 *                 to Deneb share one shape (228-byte fixed part, Bitlist[2048]); Electra adds committee_bits
 *                 (236 bytes, Bitlist[131072]).
 *   caches        1 to 3 committee caches of distinct epochs; an attestation uses the one of data.slot / 32.
 *   fork_info     domain = compute_domain(DOMAIN_BEACON_ATTESTER, previous_version if target.epoch < epoch else
 *                 current_version, genesis_validators_root) (ChainSpec::get_domain).
 *   rands         n nonzero scalars (attestation i's), or NULL to draw them like lhb200_verify_signature_sets.
 *   *ok           verify_signature_sets over the attestations whose status is 0 (0 when there is none).
 *   status        n bytes: 0 fine; LHB200_ATT_* (10-14) an indexing error, in that precedence, and the attestation is
 *                 left out of the batch; else the set's verify status (1-6, see lhb200_verify_signature_sets; an
 *                 empty index set reaches the batch and reports 4).
 *   signing_roots optional, n x 32 B (zeros for a MALFORMED record).
 *   indices_offsets, indices  optional together: the IndexedAttestation indices, sorted ascending, as a CSR
 *                 (indices_offsets: n + 1 entries) for every attestation of status 0, 1-6 or UNKNOWN_VALIDATOR (empty
 *                 for the others).  indices_cap below the total -> LHB200_EINVAL before any output is written.
 * One read-back (status, key count and signing root per attestation) lets the host group the messages and size the
 * key-index buffer; the indices then go from the committee caches straight into the batch on the device.  The launch
 * count does not depend on n or on committee sizes.  Refusals -> LHB200_EINVAL: null pointers, n == 0, non-monotone
 * offsets, a zero scalar, n_caches outside 1..3 or two caches of one epoch, an unknown fork.  Concurrent calls each
 * borrow a pooled batch handle and hold no library-wide lock. */
#define LHB200_ATT_MALFORMED 10          /* bad offset, missing delimiter, over-long bitlist, short record */
#define LHB200_ATT_NO_CACHE 11           /* no cache at data.slot's epoch (CommitteeCacheUninitialized) */
#define LHB200_ATT_NO_COMMITTEE 12       /* a committee index >= committees_per_slot (NoCommittee) */
#define LHB200_ATT_BITFIELD_LENGTH 13    /* bitlist length != committee length(s) (InvalidBitfield) */
#define LHB200_ATT_UNKNOWN_VALIDATOR 14  /* an index >= lhb200_pubkey_table_len (ValidatorUnknown) */
typedef struct {
    uint8_t previous_version[4], current_version[4];
    uint64_t epoch;
} lhb200_fork;
LHB200_API int32_t lhb200_attestations_verify(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, int32_t fork,
                                              const lhb200_committee_cache* const* caches, uint32_t n_caches,
                                              const lhb200_pubkey_table* table, const lhb200_fork* fork_info,
                                              const uint8_t genesis_validators_root[32], const uint64_t* rands,
                                              uint8_t* ok, uint8_t* status, uint8_t* signing_roots,
                                              uint64_t* indices_offsets, uint64_t* indices, uint64_t indices_cap);
/* Test hook: the final-exponentiated product (format of lhb200_bls_batch_gt) and the kernel plan (format of
 * lhb200_bls_batch_plan; gt576 or plan may be NULL) of the batch check the calling thread's last
 * lhb200_attestations_verify ran.  LHB200_EINVAL when that call verified no set. */
LHB200_API int32_t lhb200_debug_attestations_last(uint8_t gt576[576], uint32_t* plan, uint32_t n_words);
/* Every signature set of n SignedBeaconBlocks of one fork, built against a resident BeaconState and verified in one
 * batch: BlockSignatureVerifier::include_all_signatures (block_signature_verifier.rs:150-173, signature_sets.rs), the
 * call signature_verify_chain_segment, SignatureVerifiedBlock::new (n = 1) and the gossip path (n = 1,
 * LHB200_BLOCK_SKIP_PROPOSAL) make.
 *   ssz, offsets  n SignedBeaconBlock encodings of `fork`, which must be the state's fork.
 *   block_roots   n x 32: each block's root (ConsensusContext::set_current_block_root), signed by the proposal.
 *   st            an unsharded resident state advanced to the blocks' epoch.  Its fork, genesis_validators_root, slot,
 *                 validator records and current_sync_committee are read from the handle, not from the caller.
 *   caches        the committee caches of the attestations' epochs (as for lhb200_attestations_verify).
 *   table         the pubkey table; a validator index at or above min(table length, the state's validator count) is
 *                 UNKNOWN_VALIDATOR.
 *   versions      genesis_fork_version (BLS-to-execution changes, consolidations) and capella_fork_version (exits
 *                 from Deneb on, EIP-7044).
 *   rands         optional: rands[j] (nonzero) scales set j of `sets`; n_rands at least the sets the blocks contribute.
 *   *ok           1 only when every set was constructed and the batch check passed.
 *   block_status  n bytes: the code of the block's first failing set in push order, or 0.
 *   sets, *n_sets every set in push order (proposal, randao, proposer slashings, attester slashings, attestations,
 *                 exits, sync aggregate, BLS-to-execution changes, consolidations), with its status: 0, the set's
 *                 verify status 1-6, or a construction code 10-17.  A set that fails construction stays out of the
 *                 batch.
 * Domains: get_domain(epoch, type, state.fork, gvr), except exits from Deneb on (capella_fork_version), and
 * BLS-to-execution changes and consolidations (genesis_fork_version).  The proposer of a block is get_beacon_proposer_index(block.slot); a block
 * outside the state's current epoch gets SLOT_OUT_OF_BOUNDS on its proposal and RANDAO sets.  The sync aggregate's
 * keys are the current_sync_committee members' validator indices, found by matching the resident records' pubkeys
 * (the smallest index wins); an unmatched participant gives PUBKEY_DECOMPRESSION.  A BLS-to-execution change's key is
 * its from_bls_pubkey, decompressed and key-validated on the device (PublicKey::deserialize): an infinity, off-curve or
 * non-subgroup key gives PUBKEY_DECOMPRESSION.  All-zero bits with the infinity
 * signature give no set.  Deposits carry no set (block_signature_verifier.rs:169).  The caller keeps the fork-schedule
 * check (InconsistentBlockFork), which needs the ChainSpec.
 * Refusals -> LHB200_EINVAL, nothing launched: null arguments, n == 0, a fork other than the state's, a sharded state,
 * a SignedBeaconBlock whose 100-byte fixed part does not frame its message, malformed offsets or lengths in the block,
 * its body or any list a set is read from, sets_cap or n_rands below the sets the blocks contribute, a zero scalar, and
 * the committee-cache errors of lhb200_attestations_verify.  The fields no set reads (deposits, the execution payload,
 * blob commitments) are not framed here: the blocks' roots, which the caller already has, are where they are checked.
 * The launch count and the number of host synchronises depend on neither n, the number of sets nor the validator
 * count. */
#define LHB200_BSET_PROPOSAL 0
#define LHB200_BSET_RANDAO 1
#define LHB200_BSET_PROPOSER_SLASHING 2
#define LHB200_BSET_ATTESTER_SLASHING 3
#define LHB200_BSET_ATTESTATION 4
#define LHB200_BSET_EXIT 5
#define LHB200_BSET_SYNC_AGGREGATE 6
#define LHB200_BSET_BLS_CHANGE 7
#define LHB200_BSET_CONSOLIDATION 8
#define LHB200_BLOCK_INCORRECT_PROPOSER 15   /* block.proposer_index != the state's proposer (IncorrectBlockProposer) */
#define LHB200_BLOCK_SLOT_OUT_OF_BOUNDS 16   /* the block's epoch is not the state's current epoch (SlotOutOfBounds) */
#define LHB200_BLOCK_PUBKEY_DECOMPRESSION 17 /* a sync participant's key matches no validator record, or a
                                                BLS-to-execution change's key does not decode and validate */
#define LHB200_BLOCK_SKIP_PROPOSAL 1         /* include_all_signatures_except_proposal (the gossip path) */
#define LHB200_BLOCK_MAX_SETS 199            /* sets one block can contribute (mainnet preset, pre-Electra) */
typedef struct { uint8_t genesis_fork_version[4], capella_fork_version[4]; } lhb200_chain_versions;
typedef struct {
    uint32_t block;          /* index of the block in the call */
    uint16_t item;           /* index in its body list; proposer / attester slashings: 2 i + (0 | 1); else 0 */
    uint8_t kind;            /* LHB200_BSET_* */
    uint8_t status;          /* 0, the set's verify status 1-6, or a construction code 10-17 */
    uint8_t signing_root[32];
} lhb200_block_set;
LHB200_API int32_t lhb200_block_signatures_verify(const uint8_t* ssz, const uint64_t* offsets, uint32_t n, int32_t fork,
                                                  uint32_t flags, const uint8_t* block_roots, lhb200_state* st,
                                                  const lhb200_committee_cache* const* caches, uint32_t n_caches,
                                                  const lhb200_pubkey_table* table,
                                                  const lhb200_chain_versions* versions, const uint64_t* rands,
                                                  uint64_t n_rands, uint8_t* ok, uint8_t* block_status,
                                                  lhb200_block_set* sets, uint64_t sets_cap, uint64_t* n_sets);
/* Test hook: lhb200_debug_attestations_last for the calling thread's last lhb200_block_signatures_verify.  Both hooks
 * read one per-thread record, so each reports the last batch check of either call on this thread. */
LHB200_API int32_t lhb200_debug_block_signatures_last(uint8_t gt576[576], uint32_t* plan, uint32_t n_words);
/* Test hook: the kernel launches the calling thread's last lhb200_block_signatures_verify made besides its batch
 * check's (library-wide launch counter; other threads' launches meanwhile are counted too), and the host synchronises
 * it made, the batch check's result included. */
LHB200_API int32_t lhb200_debug_block_signatures_counts(uint64_t* launches, uint64_t* syncs);
/* Test hook: final-exponentiated product of the last verify as 12 x 48-byte big-endian Fp (tower order
 * c0.c0.c0 .. c1.c2.c1).  NOTE: this is the cube of the canonical GT element (3 is coprime to r). */
LHB200_API int32_t lhb200_bls_batch_gt(lhb200_bls_batch* b, uint8_t out576[576]);
/* Test hook: which kernels the last lhb200_bls_batch_verify_enqueue on `b` launched, so a test can tell which path a
 * batch size exercised.  Writes min(n_words, LHB200_PLAN_WORDS) words, indexed by LHB200_PLAN_*; the stage words
 * hold LHB200_K_* ids, 0 where the stage did not run (the sum tree of a single set). */
#define LHB200_PLAN_WORDS 24
#define LHB200_PLAN_N_SETS 0
#define LHB200_PLAN_N_SM 1                    /* SM count the launch shapes were derived from */
#define LHB200_PLAN_SIG 2
#define LHB200_PLAN_SUM 3                     /* sum of r_i sig_i */
#define LHB200_PLAN_SUM_LEVELS 4
#define LHB200_PLAN_HASH 5
#define LHB200_PLAN_KEY 6
#define LHB200_PLAN_KEY_CHUNKS 7              /* streamed upload: chunks of whole sets; 0 = one launch */
#define LHB200_PLAN_MILLER 8
#define LHB200_PLAN_MILLER_WPB 9              /* warps per block (k_miller_warp, k_miller_coop) */
#define LHB200_PLAN_MILLER_SPW 10             /* sets per warp (k_miller_warp: 1, k_miller_coop) or per thread (multi) */
#define LHB200_PLAN_MILLER_GRID 11
#define LHB200_PLAN_MILLER_ROUNDS_CAP 12      /* k_miller_coop: rounds of 30 sets per lane */
#define LHB200_PLAN_MILLER_FEW_WARPS 13       /* k_miller_coop: 1 on the few-warps branch (small batches) */
#define LHB200_PLAN_FP12_REDUCE_LEVELS 14
#define LHB200_PLAN_N_TAIL 15                 /* Miller products the final kernel folds itself */
#define LHB200_PLAN_FINAL 16
#define LHB200_PLAN_LANE_GRID 17              /* blocks of the one-thread-per-set kernels */
#define LHB200_PLAN_LANE_SETS_PER_THREAD 18   /* > 1 once the CTA cap makes them grid-stride */
#define LHB200_PLAN_LAST_MILLER 19            /* 1 if k_last_miller ran (the pair -g1, sum r sig on its own) */
#define LHB200_PLAN_GROUPS 20                 /* distinct messages the sets were grouped into; 0 = not grouped */
#define LHB200_PLAN_GROUP_SUM 21              /* the per-message key sum (grouped batches only) */
#define LHB200_PLAN_GROUP_SUM_LEVELS 22       /* levels of its segmented tree */
#define LHB200_PLAN_SEGMENTS 23               /* independent batches of a segmented pass; 0 = one batch.  The sum word
                                               * then names the per-segment signature sum, the Miller word the
                                               * one-value-per-warp variant of k_miller_warp, the final word the
                                               * per-segment tail */
#define LHB200_K_SIG_PREPARE 1
#define LHB200_K_SIG_PREPARE_WARP 2
#define LHB200_K_G2_REDUCE 3
#define LHB200_K_G2_SUM_WARP 4
#define LHB200_K_HASH_TO_G2 5
#define LHB200_K_HASH_TO_G2_PAIR 6
#define LHB200_K_HASH_TO_G2_WARP 7
#define LHB200_K_PK_AGGREGATE 8
#define LHB200_K_PK_PARTIAL_COMBINE 9
#define LHB200_K_PK_AGGREGATE_TMA 10
#define LHB200_K_PK_AGGREGATE_INDEXED 11
#define LHB200_K_MILLER_MULTI 12
#define LHB200_K_MILLER_COOP 13
#define LHB200_K_MILLER_WARP 14
#define LHB200_K_FINAL_COOP 15
#define LHB200_K_FINAL_WARP 16
#define LHB200_K_G1_GROUP_SUM 17
#define LHB200_K_G2_SEGMENT_SUM 18
#define LHB200_K_FINAL_SEGMENTS 19
LHB200_API int32_t lhb200_bls_batch_plan(const lhb200_bls_batch* b, uint32_t* out, uint32_t n_words);
LHB200_API uint64_t lhb200_bls_batch_launches(const lhb200_bls_batch* b);
/* Device time (ms) of the Miller kernel that ran (k_miller_warp, k_miller_coop or k_miller_multi) in the last completed
 * enqueue, from CUDA events recorded on the launching stream; < 0 if unavailable. */
LHB200_API float lhb200_bls_batch_dominant_kernel_ms(const lhb200_bls_batch* b);

/* TSecretKey::public_key / ::sign (crypto/bls/src/impls/blst.rs:282-298): n big-endian 32-byte scalars (< r). */
LHB200_API int32_t lhb200_sk_to_pk(const uint8_t* sk32, uint32_t n, uint8_t* pk48, uint8_t* pk96);
LHB200_API int32_t lhb200_sign(const uint8_t* sk32, const uint8_t* msg32, uint32_t n, uint8_t* sig96);
/* PublicKey::deserialize + key_validate, batch form (blst.rs:130-140; validator_pubkey_cache.rs:116-118).
 * status[i]: 0 ok, 1 infinity (rejected), 2 bad encoding / not on curve, 3 not in subgroup. */
LHB200_API int32_t lhb200_g1_decompress_validate(const uint8_t* pk48, uint32_t n, uint8_t* pk96, uint8_t* status);
/* Signature::deserialize, batch form (blst.rs:192-194): 192-byte affine out; status 0 ok, 1 infinity, 2 bad. */
LHB200_API int32_t lhb200_g2_decompress(const uint8_t* sig96, uint32_t n, uint8_t* out192, uint8_t* status);

/* ---- multi-GPU: the library's own NCCL communicator (one process per GPU; SURVEY.md §8b/§8e) ----
 * Rank 0 obtains the 128-byte id (ncclGetUniqueId) and ships it to the other ranks by any means; every rank then calls
 * lhb200_comm_init (collective).  NCCL is dlopen'ed on first use (libnccl.so.2); single-GPU users never load it.
 * The collectives below run on DEVICE buffers on the library's streams — no host hop, no torch. */
LHB200_API int32_t lhb200_comm_unique_id(uint8_t id[128]);
LHB200_API int32_t lhb200_comm_init(int32_t rank, int32_t world, const uint8_t id[128]);
LHB200_API int32_t lhb200_comm_destroy(void);
LHB200_API int32_t lhb200_comm_info(int32_t* rank, int32_t* world);
/* bls::verify_signature_sets sharded over the communicator: each rank passes its contiguous shard of the sets (an empty
 * shard is allowed); per-rank batch check + ONE ncclAllReduce(min) of the device verdicts; *ok = verdict of the whole
 * batch on every rank.  Shard with equal key counts (lighthouse_b200/parallel.py::shard_ranges_by_keys). */
LHB200_API int32_t lhb200_verify_signature_sets_collective(const uint8_t* sigs, const uint8_t* msgs, const uint8_t* pks,
                                                           const uint32_t* pk_offsets, const uint64_t* rands,
                                                           uint32_t n_sets, uint8_t* ok);
/* Staged form: ncclAllReduce(min) of a batch's device verdict, enqueued on `stream` behind verify_enqueue. */
LHB200_API int32_t lhb200_bls_batch_allreduce_verdict(lhb200_bls_batch* b, void* stream);

/* ---- aggregation surface of a crypto/bls backend (crypto/bls/src/impls/blst.rs) ----
 * TAggregateSignature::add_assign / add_assign_aggregate (blst.rs:230-237): out = sum of n compressed signatures; no
 * subgroup check (the trait's contract), infinity encodings are the identity, n == 0 -> the infinity signature;
 * LHB200_EDECODE if an encoding is malformed. */
LHB200_API int32_t lhb200_g2_aggregate(const uint8_t* sigs96, uint32_t n, uint8_t out96[96]);
/* TAggregatePublicKey::aggregate (blst.rs:178-184; generic_aggregate_public_key.rs:9-15): sum of n uncompressed keys
 * (already validated, per the trait's contract), compressed and/or uncompressed result (either may be NULL).
 * n == 0 -> LHB200_EINVAL; malformed / off-curve key -> LHB200_EDECODE. */
LHB200_API int32_t lhb200_g1_aggregate(const uint8_t* pks96, uint32_t n, uint8_t* out48, uint8_t* out96);
/* TPublicKey::deserialize_uncompressed (blst.rs:142-150), batch form: flag bits and on-curve check, no subgroup check.
 * status[i]: 0 ok, 1 infinity, 2 bad encoding / not on the curve; pk48 (optional) receives the compressed keys.
 * NOTE: lhb200_verify_signature_sets does not repeat the curve check on its explicit `pks` (blst.rs:115
 * pks_validate = false): keys must come from this call, lhb200_g1_decompress_validate or a pubkey table. */
LHB200_API int32_t lhb200_g1_deserialize_uncompressed(const uint8_t* pks96, uint32_t n, uint8_t* pk48, uint8_t* status);
/* TAggregateSignature::aggregate_verify (blst.rs:263-273): *ok = 1 iff e(g1, sig) == prod_i e(pk_i, H(m_i)) and sig is
 * in G2.  n == 0 -> *ok = 0 (generic_aggregate_signature.rs:214-216). */
LHB200_API int32_t lhb200_aggregate_verify(const uint8_t sig96[96], const uint8_t* msgs, const uint8_t* pks96, uint32_t n,
                                           uint8_t* ok);

/* Test hook (no device needed): n blinding scalars from the generator lhb200_verify_signature_sets uses when
 * `rands == NULL` — a ChaCha20 keystream keyed from getrandom(2), zeros skipped (blst.rs:46-68: rand::thread_rng). */
LHB200_API int32_t lhb200_debug_rand_scalars(uint64_t* out, uint32_t n);
/* Test hook (no device needed): the grouping of n 32-byte messages the batch uploads apply.  members (n) lists the
 * sets group by group, groups in order of first occurrence and members ascending; group g owns
 * members[group_offsets[g] .. group_offsets[g + 1]) (group_offsets: n + 1 words, *n_groups + 1 written). */
LHB200_API int32_t lhb200_debug_group_messages(const uint8_t* msgs, uint32_t n, uint32_t* members,
                                               uint32_t* group_offsets, uint32_t* n_groups);

/* Test hook: run one stage of the BLS pipeline on a single device thread so `pytest -m gpu` can compare every
 * stage with the oracle.  op: 0 expand_message_xmd(32->256), 1 hash_to_g2(32->96), 2 SSWU(u 96 -> x|y 192),
 * 3 g2_decompress(96 -> [in_subgroup, 96 recompressed], rc=DecodeStatus), 4 g2_mul(96|u64le -> 96),
 * 5 fp2 op([opcode|a|b] -> 96), 6 pairing+final_exp(g1 96|g2 96 -> 576), 7 g1 sum([n|n*96] -> 96). */
LHB200_API int32_t lhb200_debug_bls(int32_t op, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t out_len,
                                    int32_t* rc);
/* Test hook: n cases of one base-field operation on raw little-endian 32-bit limbs, one device thread per case, so
 * `pytest -m gpu` can check the carry chains of the Fp arithmetic case by case (op codes, operand layouts and the
 * 37-word result of a case in bls/fp_probe.cuh).  in: n x in_words words (the op's operand count, else EINVAL);
 * out: n x out_words words (out_words = 37). */
LHB200_API int32_t lhb200_debug_fp_batch(int32_t op, const uint32_t* in, uint32_t in_words, uint32_t n, uint32_t* out,
                                         uint32_t out_words);

#ifdef __cplusplus
}
#endif
#endif /* LHB200_H */
