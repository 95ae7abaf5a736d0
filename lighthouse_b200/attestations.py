"""Attestations verified on the device against resident committee caches and the pubkey table
(lhb200_attestations_verify): get_attesting_indices (consensus/state_processing/src/common/get_attesting_indices.rs),
indexed_attestation_signature_set (per_block_processing/signature_sets.rs:271-332) and verify_signature_sets in one
call.  The caller hands over Attestation SSZ bytes; the committee lookup, the attesting indices, the AttestationData and
signing roots and the key gather all happen on the device.
"""
import ctypes as C

import numpy as np

from . import _ffi
from ._ffi import lib, check
from .tree_hash import FORKS

# per-attestation status: 0 fine, 1-6 the set's verify status (lhb200_verify_signature_sets), then the indexing errors
OK, MALFORMED, NO_CACHE, NO_COMMITTEE, BITFIELD_LENGTH, UNKNOWN_VALIDATOR = 0, 10, 11, 12, 13, 14
STATUS_NAMES = {0: "ok", 1: "empty signature", 2: "signature decode", 3: "signature not in subgroup", 4: "no keys",
                5: "aggregate key at infinity", 6: "key decode", 10: "malformed", 11: "no cache", 12: "no committee",
                13: "bitfield length", 14: "unknown validator"}
FIXED = {False: 228, True: 236}   # fixed part of an Attestation before / from Electra


def fork_id(fork):
    return FORKS[fork] if isinstance(fork, str) else int(fork)


def fork_struct(fork_info):
    """(previous_version: 4 bytes, current_version: 4 bytes, epoch) -> lhb200_fork"""
    prev, cur, epoch = fork_info
    f = _ffi.Fork()
    f.previous_version[:] = bytes(prev)
    f.current_version[:] = bytes(cur)
    f.epoch = int(epoch)
    return f


def verify_attestations(atts, fork, caches, table, fork_info, gvr, rands=None, want_indices=False):
    """atts: Attestation SSZ encodings of one fork ("base" .. "electra" or LHB200_FORK_*); caches: 1 to 3
    committees.DeviceCommitteeCache of distinct epochs; table: bls.PubkeyTable; fork_info: (previous_version,
    current_version, epoch); gvr: genesis_validators_root; rands: one nonzero u64 per attestation, or None.
    -> (ok, statuses uint8[n], signing_roots list of n 32-byte roots, indexed: None, or per attestation its sorted
    attesting indices as uint64, empty where indexing failed)."""
    n = len(atts)
    lens = np.fromiter((len(a) for a in atts), dtype=np.uint64, count=n)
    offs = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(lens, out=offs[1:])
    ssz = np.frombuffer(b"".join(atts) or b"\0", dtype=np.uint8)
    handles = (C.c_void_p * max(len(caches), 1))(*[c._h for c in caches])
    fi = fork_struct(fork_info)
    ok = C.c_uint8(0)
    st = np.zeros(max(n, 1), dtype=np.uint8)
    roots = np.zeros(max(n, 1) * 32, dtype=np.uint8)
    r = None if rands is None else np.ascontiguousarray(rands, dtype=np.uint64)
    fid = fork_id(fork)
    idx_off = idx = None
    cap = 0
    if want_indices:
        # every attesting index is one bit of a bitlist: the bitlist bytes bound them
        cap = max(1, 8 * int(np.maximum(lens.astype(np.int64) - FIXED[fid >= FORKS["electra"]], 0).sum()))
        idx_off = np.zeros(n + 1, dtype=np.uint64)
        idx = np.zeros(cap, dtype=np.uint64)
    check(lib.lhb200_attestations_verify(ssz.ctypes.data, offs.ctypes.data, n, fid, C.cast(handles, C.c_void_p),
                                         len(caches), table._h, C.byref(fi), bytes(gvr),
                                         None if r is None else r.ctypes.data, C.byref(ok), st.ctypes.data,
                                         roots.ctypes.data, None if idx_off is None else idx_off.ctypes.data,
                                         None if idx is None else idx.ctypes.data, cap),
          "lhb200_attestations_verify")
    raw = roots.tobytes()
    signing_roots = [raw[32 * i:32 * i + 32] for i in range(n)]
    indexed = None
    if want_indices:
        indexed = [idx[int(idx_off[i]):int(idx_off[i + 1])].copy() for i in range(n)]
    return ok.value == 1, st[:n].copy(), signing_roots, indexed


def last_batch_check():
    """Test hook (lhb200_debug_attestations_last): (gt bytes, plan dict) of the batch check the calling thread's last
    verify_attestations ran."""
    from .bls import PLAN_FIELDS, PLAN_KERNELS, _PLAN_KERNEL_FIELDS
    gt = C.create_string_buffer(576)
    w = np.zeros(len(PLAN_FIELDS), dtype=np.uint32)
    check(lib.lhb200_debug_attestations_last(gt, w.ctypes.data, len(w)), "lhb200_debug_attestations_last")
    plan = {f: (PLAN_KERNELS[int(v)] if f in _PLAN_KERNEL_FIELDS else int(v)) for f, v in zip(PLAN_FIELDS, w)}
    return gt.raw, plan
