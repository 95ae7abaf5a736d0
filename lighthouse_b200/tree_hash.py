"""Host-side mirror of the tree_hash / ethereum_hashing surface Lighthouse's types call
(tree_hash::{merkle_root, mix_in_length, BYTES_PER_CHUNK}, ethereum_hashing::{hash32_concat, ZERO_HASHES},
BeaconState::update_tree_hash_cache — /root/reference/consensus/types/src/beacon_state.rs:2031-2038).
Every function dispatches to the CUDA library through the C ABI; there is no CPU arithmetic here.
"""
import ctypes as C

from . import _ffi
from ._ffi import lib, check, buf

BYTES_PER_CHUNK = 32
HASHSIZE = 32
VALIDATOR_SSZ_BYTES = 121


def hash32_concat(a: bytes, b: bytes) -> bytes:
    assert len(a) == 32 and len(b) == 32
    return hash_pairs(a + b)


def hash_pairs(data: bytes) -> bytes:
    """n x 64 bytes -> n x 32 bytes (batch of ethereum_hashing::hash32_concat)."""
    assert len(data) % 64 == 0
    n = len(data) // 64
    out = C.create_string_buffer(max(n * 32, 1))
    p, keep = buf(data)
    check(lib.lhb200_hash_pairs(p, out, n), "lhb200_hash_pairs")
    return out.raw[: n * 32]


def zero_hash(depth: int) -> bytes:
    out = C.create_string_buffer(32)
    check(lib.lhb200_zero_hash(depth, out), "lhb200_zero_hash")
    return out.raw


def merkleize_chunks(chunks: bytes, depth: int) -> bytes:
    """merkleize(chunks, limit = 2**depth)."""
    assert len(chunks) % 32 == 0
    out = C.create_string_buffer(32)
    p, keep = buf(chunks)
    check(lib.lhb200_merkleize(p, len(chunks) // 32, depth, out), "lhb200_merkleize")
    return out.raw


def merkle_root(data: bytes, minimum_leaf_count: int = 0) -> bytes:
    """tree_hash::merkle_root(bytes, minimum_leaf_count): zero-pad to whole chunks, tree height from
    max(next_pow2(#chunks), next_pow2(minimum_leaf_count)) (used at crypto/bls/src/macros.rs:24)."""
    n = max((len(data) + 31) // 32, 1)
    padded = data + b"\0" * (n * 32 - len(data))
    leaves = max(n, minimum_leaf_count, 1)
    depth = (leaves - 1).bit_length()
    return merkleize_chunks(padded, depth)


class MerkleHasher:
    """tree_hash::MerkleHasher {with_leaves, write, finish} as used by AttestationKey::tree_hash_root
    (beacon_node/beacon_chain/src/naive_aggregation_pool.rs:46-55): written bytes are concatenated, cut into 32-byte
    leaves (the last one zero-padded at finish) and merkleized over `num_leaves`.  The crate (tree_hash 0.6.0) is not
    vendored; the only in-tree call site writes a 32-byte root then an 8-byte index, where this is unambiguous."""

    def __init__(self, num_leaves: int):
        self.num_leaves = max(int(num_leaves), 1)
        self._chunks = bytearray()

    @classmethod
    def with_leaves(cls, num_leaves: int):
        return cls(num_leaves)

    def write(self, data: bytes):
        data = bytes(data)
        if len(self._chunks) + len(data) > 32 * self.num_leaves:
            raise ValueError("MerkleHasher: MaximumLeavesExceeded")
        self._chunks += data
        return self

    def finish(self) -> bytes:
        depth = (self.num_leaves - 1).bit_length()
        data = bytes(self._chunks)
        return merkleize_chunks(data + b"\0" * (-len(data) % 32), depth)


def mix_in_length(root: bytes, length: int) -> bytes:
    out = C.create_string_buffer(32)
    p, keep = buf(root)
    check(lib.lhb200_mix_in_length(p, length, out), "lhb200_mix_in_length")
    return out.raw


def validators_root(ssz: bytes) -> bytes:
    """hash_tree_root(List[Validator, 2**40]) from concatenated 121-byte SSZ validators."""
    assert len(ssz) % VALIDATOR_SSZ_BYTES == 0
    out = C.create_string_buffer(32)
    p, keep = buf(ssz)
    check(lib.lhb200_validators_root(p, len(ssz) // VALIDATOR_SSZ_BYTES, out), "lhb200_validators_root")
    return out.raw


def validator_roots(ssz: bytes) -> bytes:
    n = len(ssz) // VALIDATOR_SSZ_BYTES
    out = C.create_string_buffer(max(32 * n, 1))
    p, keep = buf(ssz)
    check(lib.lhb200_validator_roots(p, n, out), "lhb200_validator_roots")
    return out.raw[: 32 * n]


FORKS = {"base": 0, "altair": 1, "bellatrix": 2, "capella": 3, "deneb": 4, "electra": 5}   # LHB200_FORK_*


def _n_field_roots(fork):
    """Field roots the state entry points write: 28 for every fork before Electra (zero chunks past the fork's own
    fields), 37 for Electra."""
    return 37 if fork == "electra" else 28


def beacon_state_root_deneb(ssz, want_field_roots=False):
    """BeaconState::update_tree_hash_cache (cold) for BeaconStateDeneb SSZ bytes."""
    return beacon_state_root(ssz, "deneb", want_field_roots)


def beacon_state_root(ssz, fork="deneb", want_field_roots=False):
    """BeaconState::update_tree_hash_cache (cold) for any variant of the superstruct from Base (phase0) on
    (consensus/types/src/beacon_state.rs:224-571): lhb200_beacon_state_root."""
    out = C.create_string_buffer(32)
    n_fr = _n_field_roots(fork)
    fr = C.create_string_buffer(n_fr * 32) if want_field_roots else None
    p, keep = buf(ssz)
    n = len(ssz) if isinstance(ssz, (bytes, bytearray)) else keep.nbytes
    check(lib.lhb200_beacon_state_root(p, n, FORKS[fork], out, fr), "lhb200_beacon_state_root")
    if want_field_roots:
        return out.raw, [fr.raw[32 * i: 32 * i + 32] for i in range(n_fr)]
    return out.raw


def beacon_block_roots_deneb(blocks, want_body_roots=False, blinded=False):
    """BeaconBlock::canonical_root (beacon_block.rs:158-160) of a batch of BeaconBlockDeneb SSZ blobs in one pass
    (blinded=True: BlindedBeaconBlockDeneb blobs, whose body carries the payload header)."""
    return beacon_block_roots(blocks, "deneb", want_body_roots, blinded)


def beacon_block_roots(blocks, fork="deneb", want_body_roots=False, blinded=False):
    """canonical_root of a batch of BeaconBlock<fork> (or BlindedBeaconBlock<fork>) SSZ blobs, fork in base / altair /
    bellatrix / capella / deneb / electra (beacon_block.rs:19-90; no blinded Base form): lhb200_beacon_block_roots."""
    blocks = [bytes(b) for b in blocks]
    n = len(blocks)
    offs = (C.c_uint64 * (n + 1))()
    for i, b in enumerate(blocks):
        offs[i + 1] = offs[i] + len(b)
    p, keep = buf(b"".join(blocks))
    out = C.create_string_buffer(32 * max(n, 1))
    body = C.create_string_buffer(32 * max(n, 1)) if want_body_roots else None
    check(lib.lhb200_beacon_block_roots(p, C.cast(offs, C.c_void_p), n, FORKS[fork], 1 if blinded else 0, out, body),
          "lhb200_beacon_block_roots")
    roots = [out.raw[32 * i: 32 * i + 32] for i in range(n)]
    if want_body_roots:
        return roots, [body.raw[32 * i: 32 * i + 32] for i in range(n)]
    return roots


# Generalized indices the reference proves (light_client_update.rs, beacon_block_body.rs; consensus-specs
# ssz/merkle-proofs.md).  The state ones are for the 32-leaf top tree of Altair to Deneb; Electra's 37 fields take a
# 64-leaf top tree, one level deeper.
FINALIZED_ROOT_INDEX = 105            # finalized_checkpoint.root: (32 + 20) * 2 + 1
CURRENT_SYNC_COMMITTEE_INDEX = 54
NEXT_SYNC_COMMITTEE_INDEX = 55
FINALIZED_ROOT_INDEX_ELECTRA = 169    # (64 + 20) * 2 + 1
CURRENT_SYNC_COMMITTEE_INDEX_ELECTRA = 86
NEXT_SYNC_COMMITTEE_INDEX_ELECTRA = 87
EXECUTION_PAYLOAD_INDEX = 25          # body field 9 of a 16-leaf body tree (Bellatrix to Electra)
BLOB_KZG_COMMITMENTS_INDEX = 27       # body field 11
KZG_COMMITMENT_INCLUSION_PROOF_DEPTH = 17


def kzg_commitment_gindex(i):
    """Body gindex of blob_kzg_commitments[i]: field 27, the list's data root (27 * 2), then depth 12 (4096 items)."""
    return 54 * 4096 + i


def _split_branches(g, call, where, raw):
    """Run `call(out, root)` for the gindices g (uint64 array) and cut the flat output into per-proof branches."""
    import numpy as np
    depths = np.array([int(x).bit_length() - 1 if x else 0 for x in g.tolist()], dtype=np.int64)
    total = int(depths.sum())
    out = np.zeros(max(32 * total, 1), dtype=np.uint8)
    root = C.create_string_buffer(32)
    check(call(C.c_void_p(out.ctypes.data), root), where)
    if raw:
        return root.raw, out[:32 * total]
    flat, at, branches = out.tobytes(), 0, []
    for d in depths.tolist():
        branches.append([flat[32 * (at + k): 32 * (at + k + 1)] for k in range(d)])
        at += d
    return root.raw, branches


def beacon_block_body_proofs(blocks, proofs, fork="deneb", blinded=False, raw=False):
    """Merkle branches below the BODY roots of a batch of BeaconBlock<fork> (or blinded) SSZ blobs, in one pass
    (lhb200_beacon_block_body_proofs).  proofs: [(block index, body gindex), ...].  -> (body roots, branches), branches
    as ResidentState.proofs gives them (kzg_commitment_gindex(i): the 17-sibling blob inclusion proof)."""
    import numpy as np
    blocks = [bytes(b) for b in blocks]
    n = len(blocks)
    offs = (C.c_uint64 * (n + 1))()
    for i, b in enumerate(blocks):
        offs[i + 1] = offs[i] + len(b)
    p, keep = buf(b"".join(blocks))
    block_of = np.ascontiguousarray([b for b, _ in proofs], dtype=np.uint32)
    g = np.ascontiguousarray([x for _, x in proofs], dtype=np.uint64)
    body = C.create_string_buffer(32 * max(n, 1))
    root, branches = _split_branches(g, lambda out, _root: lib.lhb200_beacon_block_body_proofs(
        p, C.cast(offs, C.c_void_p), n, FORKS[fork], 1 if blinded else 0, block_of.ctypes.data, g.ctypes.data, len(g),
        out, body), "lhb200_beacon_block_body_proofs", raw)
    return [body.raw[32 * i: 32 * i + 32] for i in range(n)], branches


def debug_proof_gather_ms():
    """Benchmark hook: device time of the last k_proof_branches launch (CUDA events), < 0 if unavailable."""
    return float(lib.lhb200_debug_proof_gather_ms())


def beacon_block_root_deneb(ssz, want_body_root=False, blinded=False):
    """canonical_root of one BeaconBlockDeneb; optionally also hash_tree_root(body) (BeaconBlockHeader.body_root)."""
    r = beacon_block_roots_deneb([ssz], want_body_root, blinded)
    return (r[0][0], r[1][0]) if want_body_root else r[0]


class ShardedState:
    """One rank's shard of a BeaconStateDeneb hashed over `world` GPUs (SURVEY.md §8e)."""

    def __init__(self, ssz, rank, world):
        self._h = C.c_void_p()
        p, keep = buf(ssz)
        n = len(ssz) if isinstance(ssz, (bytes, bytearray)) else keep.nbytes
        check(lib.lhb200_state_stage_deneb_shard(p, n, rank, world, C.byref(self._h)), "lhb200_state_stage_deneb_shard")
        self.world = world

    def shard_roots(self) -> bytes:
        out = C.create_string_buffer(32 * 16)
        n = C.c_uint32(0)
        check(lib.lhb200_state_shard_roots(self._h, out, C.byref(n)), "lhb200_state_shard_roots")
        return out.raw[: 32 * n.value]

    def combine(self, gathered: bytes) -> bytes:
        out = C.create_string_buffer(32)
        p, keep = buf(gathered)
        check(lib.lhb200_state_combine(self._h, p, out), "lhb200_state_combine")
        return out.raw

    def root_collective(self, stream=None) -> bytes:
        """lhb200_state_root_sharded: shard roots -> ncclAllGather (library communicator) -> combine, all on the device."""
        out = C.create_string_buffer(32)
        check(lib.lhb200_state_root_sharded(self._h, out), "lhb200_state_root_sharded")
        return out.raw

    def release(self):
        if self._h:
            lib.lhb200_state_release(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class ResidentState:
    """A BeaconState staged once into HBM (DESIGN.md §3) and hashed from there.  `fork` in base / altair / bellatrix /
    capella / deneb / electra; Deneb stages through lhb200_state_stage_deneb, the others through lhb200_state_stage."""

    def __init__(self, ssz, fork="deneb"):
        self._h = C.c_void_p()
        self.fork = fork
        p, keep = buf(ssz)
        n = len(ssz) if isinstance(ssz, (bytes, bytearray)) else keep.nbytes
        if fork == "deneb":
            check(lib.lhb200_state_stage_deneb(p, n, C.byref(self._h)), "lhb200_state_stage_deneb")
        else:
            check(lib.lhb200_state_stage(p, n, FORKS[fork], C.byref(self._h)), "lhb200_state_stage")

    def root(self, want_field_roots=False):
        out = C.create_string_buffer(32)
        n_fr = _n_field_roots(self.fork)
        fr = C.create_string_buffer(n_fr * 32) if want_field_roots else None
        check(lib.lhb200_state_root(self._h, out, fr), "lhb200_state_root")
        if want_field_roots:
            return out.raw, [fr.raw[32 * i: 32 * i + 32] for i in range(n_fr)]
        return out.raw

    def patch(self, ssz_offset: int, data: bytes):
        """Same-length mutation of SSZ bytes [ssz_offset, ssz_offset + len(data)) (apply_pending_mutations)."""
        p, keep = buf(data)
        check(lib.lhb200_state_patch(self._h, ssz_offset, p, len(data)), "lhb200_state_patch")

    def patch_batch(self, edits):
        """[(ssz_offset, bytes), ...] non-overlapping same-length mutations in one call (one copy + one scatter kernel)."""
        import numpy as np
        edits = list(edits)
        if not edits:
            return
        offs = np.array([o for o, _ in edits], dtype=np.uint64)
        lens = np.array([len(d) for _, d in edits], dtype=np.uint32)
        p, keep = buf(b"".join(d for _, d in edits))
        check(lib.lhb200_state_patch_batch(self._h, offs.ctypes.data, lens.ctypes.data, p, len(edits)),
              "lhb200_state_patch_batch")

    def enable_incremental(self):
        """Warm path: keep every level of the big lists resident; later root() calls re-hash only the paths above
        the leaves patch() touched (the reference's tree-hash-cache behaviour, beacon_state.rs:2031-2038)."""
        check(lib.lhb200_state_enable_incremental(self._h), "lhb200_state_enable_incremental")

    def _list_field(self, field):
        """(container index, item bytes) of a resizable list named as in ssz_schema (or given by index)."""
        from .ssz_schema import BEACON_STATE_BY_FORK, fixed_size
        fields = BEACON_STATE_BY_FORK[self.fork][1]
        idx = field if isinstance(field, int) else [name for name, _ in fields].index(field)
        t = fields[idx][1]
        return idx, (fixed_size(t[1]) if t[0] == "list" else 0)

    def list_edit(self, edits):
        """Resize and write lists in one call (lhb200_state_list_edit): [(field, new_len, first, items_ssz), ...], at most
        one edit per field; items_ssz holds the SSZ bytes of items [first, first + n).  Needs enable_incremental()."""
        edits = list(edits)
        arr = (_ffi.ListEdit * max(len(edits), 1))()
        blobs = []
        for i, (field, new_len, first, data) in enumerate(edits):
            idx, item = self._list_field(field)
            data = bytes(data)
            if item == 0 or len(data) % item:
                raise ValueError(f"{field}: not a list of fixed-size items, or {len(data)} bytes is not whole items")
            arr[i] = _ffi.ListEdit(idx, 0, new_len, first, len(data) // item)
            blobs.append(data)
        p, keep = buf(b"".join(blobs))
        check(lib.lhb200_state_list_edit(self._h, C.cast(arr, C.c_void_p), len(edits), p), "lhb200_state_list_edit")

    def append(self, field, items_ssz):
        """Append the SSZ items to list `field` (a deposit, an eth1 vote, a historical summary, ...)."""
        n = self.list_len(field)
        _, item = self._list_field(field)
        self.list_edit([(field, n + len(items_ssz) // max(item, 1), n, items_ssz)])

    def truncate(self, field, new_len):
        """Shorten list `field` to new_len items (0: reset)."""
        self.list_edit([(field, new_len, new_len, b"")])

    def list_len(self, field):
        idx, _ = self._list_field(field)
        n = C.c_uint64(0)
        check(lib.lhb200_state_list_len(self._h, idx, C.byref(n)), "lhb200_state_list_len")
        return n.value

    def set_payload_header(self, ssz):
        """Replace latest_execution_payload_header with SSZ of this fork's header (extra_data may change length)."""
        p, keep = buf(ssz)
        check(lib.lhb200_state_set_payload_header(self._h, p, len(ssz)), "lhb200_state_set_payload_header")

    def set_pending_attestations(self, name, ssz):
        """Base: replace previous_epoch_attestations or current_epoch_attestations (by name or field index 15 / 16)
        with the SSZ of a List[PendingAttestation, 4096] (lhb200_state_set_pending_attestations).  A block appends to
        the current list; the epoch rotation is two calls.  Needs enable_incremental()."""
        idx = name if isinstance(name, int) else {"previous_epoch_attestations": 15, "current_epoch_attestations": 16}[name]
        p, keep = buf(ssz)
        check(lib.lhb200_state_set_pending_attestations(self._h, idx, p, len(ssz)), "lhb200_state_set_pending_attestations")

    def clone(self):
        """BeaconState::clone on the device (lhb200_state_clone): a new handle of the same fork whose device memory is
        its own, with this one's pending mutations; edits, roots and release of either never affect the other."""
        new = ResidentState.__new__(ResidentState)
        new._h = C.c_void_p()
        new.fork = self.fork
        check(lib.lhb200_state_clone(self._h, C.byref(new._h)), "lhb200_state_clone")
        return new

    def proofs(self, gindices, raw=False):
        """Merkle branches of generalized indices of this state, in one call (lhb200_state_proofs): roots the handle
        first, as root() does.  -> (state root, branches): branch i lists floor(log2(gindices[i])) 32-byte siblings,
        bottom-up.  raw=True returns the branches as one flat uint8 array (proof i at 32 * the depths before it)."""
        import numpy as np
        g = np.ascontiguousarray(np.asarray(gindices, dtype=np.uint64).reshape(-1))
        return _split_branches(g, lambda out, root: lib.lhb200_state_proofs(self._h, g.ctypes.data, len(g), out, root),
                               "lhb200_state_proofs", raw)

    def compute_merkle_proof(self, gindex):
        """BeaconState::compute_merkle_proof (beacon_state.rs:2483) by the spec's generalized index: the branch."""
        return self.proofs([gindex])[1][0]

    def committee_cache(self, epoch):
        """CommitteeCache::initialized(state, epoch) on the device (lhb200_state_committee_cache) -> a
        committees.CommitteeCache.  Refused (Lhb200Error, EINVAL): an epoch out of bounds, no active validator, a
        sharded handle.  The handle is only read."""
        import numpy as np
        from .committees import CommitteeCache
        n = self.list_len("validators")
        shuffling = np.zeros(max(n, 1), dtype=np.uint64)
        positions = np.zeros(max(n, 1), dtype=np.uint32)
        info = _ffi.CommitteeInfo()
        check(lib.lhb200_state_committee_cache(self._h, epoch, shuffling.ctypes.data, positions.ctypes.data, n,
                                               C.byref(info)), "lhb200_state_committee_cache")
        return CommitteeCache(info.epoch, shuffling[:info.n_active], positions[:n], info.committees_per_slot,
                              bytes(info.seed))

    def device_committee_cache(self, epoch):
        """The same cache left on the device (lhb200_state_committee_cache_create) -> a
        committees.DeviceCommitteeCache, independent of this handle once made.  Refused as committee_cache is."""
        from .committees import DeviceCommitteeCache
        h = C.c_void_p()
        check(lib.lhb200_state_committee_cache_create(self._h, epoch, C.byref(h)), "lhb200_state_committee_cache_create")
        return DeviceCommitteeCache(h)

    def beacon_proposer_indices(self):
        """BeaconState::get_beacon_proposer_indices: the proposer of each of the current epoch's 32 slots."""
        out = (C.c_uint64 * 32)()
        check(lib.lhb200_state_beacon_proposer_indices(self._h, out), "lhb200_state_beacon_proposer_indices")
        return list(out)

    def next_sync_committee_indices(self):
        """BeaconState::get_next_sync_committee_indices: 512 validator indices, duplicates kept."""
        out = (C.c_uint64 * 512)()
        check(lib.lhb200_state_next_sync_committee_indices(self._h, out), "lhb200_state_next_sync_committee_indices")
        return list(out)

    @property
    def device_bytes(self):
        """HBM the handle holds (lhb200_state_device_bytes)."""
        n = C.c_uint64(0)
        check(lib.lhb200_state_device_bytes(self._h, C.byref(n)), "lhb200_state_device_bytes")
        return n.value

    @property
    def last_root_hashes(self):
        """hash32_concat units the last root() actually computed (cold: all of them; warm: dirty paths + tail)."""
        return lib.lhb200_state_last_root_hashes(self._h)

    def enqueue(self, stream=None):
        d = C.c_void_p()
        check(lib.lhb200_state_root_enqueue(self._h, stream, C.byref(d)), "lhb200_state_root_enqueue")
        return d.value

    @property
    def hash_units(self):
        return lib.lhb200_state_hash_units(self._h)

    @property
    def dominant_kernel_ms(self):
        return float(lib.lhb200_state_dominant_kernel_ms(self._h))

    def release(self):
        if self._h:
            lib.lhb200_state_release(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


# ---- SignedRoot / domain helpers (consensus/types/src/signing_data.rs:27-35, chain_spec.rs:518-566) ----------
def container_root(field_roots) -> bytes:
    """merkleize(field roots, next_pow2(#fields)) — what #[derive(TreeHash)] emits for a container."""
    k = len(field_roots)
    depth = (max(k, 1) - 1).bit_length()
    return merkleize_chunks(b"".join(field_roots), depth)


def compute_fork_data_root(current_version: bytes, genesis_validators_root: bytes) -> bytes:
    assert len(current_version) == 4 and len(genesis_validators_root) == 32
    return hash32_concat(current_version + bytes(28), genesis_validators_root)


def compute_domain(domain_type: int, fork_version: bytes, genesis_validators_root: bytes) -> bytes:
    """ChainSpec::compute_domain: le32(domain_type) || fork_data_root[:28]"""
    return domain_type.to_bytes(4, "little") + compute_fork_data_root(fork_version, genesis_validators_root)[:28]


def signing_roots(object_roots: bytes, domain: bytes) -> bytes:
    """Batch SignedRoot::signing_root: n x 32-byte object roots -> n x 32-byte signing roots, one launch."""
    assert len(object_roots) % 32 == 0 and len(domain) == 32
    n = len(object_roots) // 32
    pairs = b"".join(object_roots[32 * i:32 * i + 32] + domain for i in range(n))
    return hash_pairs(pairs)
