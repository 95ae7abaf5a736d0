"""Every signature set of SignedBeaconBlocks built against a resident BeaconState and verified in one device batch
(lhb200_block_signatures_verify): BlockSignatureVerifier::include_all_signatures
(consensus/state_processing/src/per_block_processing/block_signature_verifier.rs:150-173) with the sets of
signature_sets.rs, as signature_verify_chain_segment, SignatureVerifiedBlock::new and the gossip path
(skip_proposal=True) call it.  The caller hands over SignedBeaconBlock SSZ bytes and the blocks' roots; the proposers,
sync-committee keys, signing roots, attesting indices and key gather all happen on the device.
"""
import ctypes as C

import numpy as np

from . import _ffi
from ._ffi import lib, check
from .attestations import fork_id

# set kinds, in push order
PROPOSAL, RANDAO, PROPOSER_SLASHING, ATTESTER_SLASHING, ATTESTATION, EXIT, SYNC_AGGREGATE, BLS_CHANGE, CONSOLIDATION = \
    range(9)
KIND_NAMES = ("proposal", "randao", "proposer_slashing", "attester_slashing", "attestation", "exit", "sync_aggregate",
              "bls_change", "consolidation")
# construction codes after the attestation codes 10-14 (lighthouse_b200.attestations)
INCORRECT_PROPOSER, SLOT_OUT_OF_BOUNDS, PUBKEY_DECOMPRESSION = 15, 16, 17
SKIP_PROPOSAL = 1
MAX_SETS_PER_BLOCK = 199


def chain_versions(genesis_fork_version, capella_fork_version):
    v = _ffi.ChainVersions()
    v.genesis_fork_version[:] = bytes(genesis_fork_version)
    v.capella_fork_version[:] = bytes(capella_fork_version)
    return v


def verify_block_signatures(blocks, fork, state, caches, table, versions, block_roots, rands=None, skip_proposal=False):
    """blocks: SignedBeaconBlock SSZ encodings of one fork ("base" .. "electra" or LHB200_FORK_*), the fork of `state`
    (a tree_hash.ResidentState advanced to the blocks' epoch); caches: 1 to 3 committees.DeviceCommitteeCache of
    distinct epochs; table: bls.PubkeyTable; versions: (genesis_fork_version, capella_fork_version); block_roots: one
    32-byte root per block; rands: one nonzero u64 per set in push order, or None.
    -> (ok, block_status uint8[n], sets: list of (block, item, kind, status, signing_root) in push order)."""
    n = len(blocks)
    lens = np.fromiter((len(b) for b in blocks), dtype=np.uint64, count=n)
    offs = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(lens, out=offs[1:])
    ssz = np.frombuffer(b"".join(blocks) or b"\0", dtype=np.uint8)
    roots = np.frombuffer(b"".join(bytes(r) for r in block_roots) or bytes(32), dtype=np.uint8)
    handles = (C.c_void_p * max(len(caches), 1))(*[c._h for c in caches])
    vs = chain_versions(*versions)
    r = None if rands is None else np.ascontiguousarray(rands, dtype=np.uint64)
    cap = max(1, n * MAX_SETS_PER_BLOCK + 16 * n)   # Electra: + 1 consolidation; never below what a block can hold
    out = (_ffi.BlockSet * cap)()
    ok = C.c_uint8(0)
    st = np.zeros(max(n, 1), dtype=np.uint8)
    n_sets = C.c_uint64(0)
    check(lib.lhb200_block_signatures_verify(ssz.ctypes.data, offs.ctypes.data, n, fork_id(fork),
                                             SKIP_PROPOSAL if skip_proposal else 0, roots.ctypes.data, state._h,
                                             C.cast(handles, C.c_void_p), len(caches), table._h, C.byref(vs),
                                             None if r is None else r.ctypes.data, 0 if r is None else len(r),
                                             C.byref(ok), st.ctypes.data, out, cap, C.byref(n_sets)),
          "lhb200_block_signatures_verify")
    sets = [(int(s.block), int(s.item), int(s.kind), int(s.status), bytes(s.signing_root))
            for s in out[:n_sets.value]]
    return ok.value == 1, st[:n].copy(), sets


def last_batch_check():
    """Test hook (lhb200_debug_block_signatures_last): (gt bytes, plan dict) of the batch check the calling thread's
    last verify_block_signatures ran."""
    from .bls import PLAN_FIELDS, PLAN_KERNELS, _PLAN_KERNEL_FIELDS
    gt = C.create_string_buffer(576)
    w = np.zeros(len(PLAN_FIELDS), dtype=np.uint32)
    check(lib.lhb200_debug_block_signatures_last(gt, w.ctypes.data, len(w)), "lhb200_debug_block_signatures_last")
    plan = {f: (PLAN_KERNELS[int(v)] if f in _PLAN_KERNEL_FIELDS else int(v)) for f, v in zip(PLAN_FIELDS, w)}
    return gt.raw, plan


def last_counts():
    """Test hook (lhb200_debug_block_signatures_counts): (launches besides the batch check's, host synchronises) of
    the calling thread's last verify_block_signatures."""
    la, sy = C.c_uint64(0), C.c_uint64(0)
    check(lib.lhb200_debug_block_signatures_counts(C.byref(la), C.byref(sy)), "lhb200_debug_block_signatures_counts")
    return la.value, sy.value
