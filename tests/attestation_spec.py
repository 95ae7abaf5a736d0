"""From-spec restatement of attestation indexing and signing roots (no GPU): both forms of get_attesting_indices
(consensus/state_processing/src/common/get_attesting_indices.rs) over the committees of tests/committee_spec.py, the
AttestationData root, compute_domain and the signing root (signature_sets.rs:271-332, ChainSpec::get_domain), and the
statuses lhb200_attestations_verify reports for the errors the reference raises before the signature check, in the
order it raises them.  hashlib and numpy only."""
import hashlib
import struct

import numpy as np

from tests import committee_spec as CS

OK, MALFORMED, NO_CACHE, NO_COMMITTEE, BITFIELD_LENGTH, UNKNOWN_VALIDATOR = 0, 10, 11, 12, 13, 14
DOMAIN_BEACON_ATTESTER = 1
FIXED = {False: 228, True: 236}
MAX_BITS = {False: 2048, True: 131072}


def sha(b):
    return hashlib.sha256(b).digest()


def spec_cache(c):
    """A committee_spec.committee_cache dict, or a committees.CommitteeCache -> (epoch, shuffling, committees_per_slot)"""
    if isinstance(c, dict):
        return c["epoch"], np.asarray(c["shuffling"], dtype=np.uint64), c["committees_per_slot"]
    return c.initialized_epoch, np.asarray(c.shuffling(), dtype=np.uint64), c.committees_per_slot()


def parse(ssz, electra):
    """-> dict(data, signature, bits (uint8 array), committee_bits) or None when the encoding is malformed: a short
    record, an offset that does not point right behind the fixed part, no delimiter, too many bits."""
    fixed = FIXED[electra]
    if len(ssz) < fixed + 1 or struct.unpack_from("<I", ssz, 0)[0] != fixed:
        return None
    raw = np.frombuffer(ssz[fixed:], dtype=np.uint8)
    if raw[-1] == 0:
        return None
    bits = np.unpackbits(raw, bitorder="little")
    n_bits = len(bits) - 8 + int(raw[-1]).bit_length() - 1
    if n_bits > MAX_BITS[electra]:
        return None
    return {"data": bytes(ssz[4:132]), "signature": bytes(ssz[132:228]), "bits": bits[:n_bits],
            "committee_bits": struct.unpack_from("<Q", ssz, 228)[0] if electra else None}


def attestation_data_root(data):
    """hash_tree_root(AttestationData {slot, index, beacon_block_root, source, target}): 8 leaves."""
    def leaf(b):
        return b + bytes(32 - len(b))
    slot, index, bbr = leaf(data[0:8]), leaf(data[8:16]), data[16:48]
    source = sha(leaf(data[48:56]) + data[56:88])
    target = sha(leaf(data[88:96]) + data[96:128])
    z = bytes(32)
    return sha(sha(sha(slot + index) + sha(bbr + source)) + sha(sha(target + z) + sha(z + z)))


def compute_domain(domain_type, version, gvr):
    return domain_type.to_bytes(4, "little") + sha(bytes(version) + bytes(28) + bytes(gvr))[:28]


def signing_root(data, fork_info, gvr):
    """signing_root(data, get_domain(target.epoch, BeaconAttester, fork, gvr))"""
    prev, cur, fork_epoch = fork_info
    target_epoch = struct.unpack_from("<Q", data, 88)[0]
    domain = compute_domain(DOMAIN_BEACON_ATTESTER, prev if target_epoch < fork_epoch else cur, gvr)
    return sha(attestation_data_root(data) + domain)


def committee(epoch_shuffling_cps, slot, index):
    _, shuffling, cps = epoch_shuffling_cps
    count = cps * CS.SLOTS_PER_EPOCH
    lo, hi = CS.committee_range(count, (slot % CS.SLOTS_PER_EPOCH) * cps + index, len(shuffling))
    return shuffling[lo:hi]


def get_attesting_indices(att, electra, caches):
    """-> (status, sorted uint64 indices or None).  The cache of data.slot's epoch (else NO_CACHE, the reference's
    uninitialised cache); before Electra the committee data.index (NO_COMMITTEE at or beyond committees_per_slot) and a
    bitlist of its length (BITFIELD_LENGTH); in Electra the committee_bits committees in ascending order (the first at
    or beyond committees_per_slot: NO_COMMITTEE), then the bitlist length against their summed lengths."""
    slot = struct.unpack_from("<Q", att["data"], 0)[0]
    cache = next((c for c in map(spec_cache, caches) if c[0] == slot // CS.SLOTS_PER_EPOCH), None)
    if cache is None:
        return NO_CACHE, None
    cps, bits = cache[2], att["bits"]
    if not electra:
        index = struct.unpack_from("<Q", att["data"], 8)[0]
        if index >= cps:
            return NO_COMMITTEE, None
        members = committee(cache, slot, index)
        if len(bits) != len(members):
            return BITFIELD_LENGTH, None
        return OK, np.sort(members[bits == 1])
    out, offset = [], 0
    for index in [k for k in range(64) if (att["committee_bits"] >> k) & 1]:
        if index >= cps:
            return NO_COMMITTEE, None
        members = committee(cache, slot, index)
        seg = bits[offset:offset + len(members)]
        out.append(members[:len(seg)][seg == 1])
        offset += len(members)
    if offset != len(bits):
        return BITFIELD_LENGTH, None
    return OK, np.sort(np.concatenate(out)) if out else np.zeros(0, dtype=np.uint64)


def index_attestation(ssz, electra, caches, table_len, fork_info, gvr):
    """What lhb200_attestations_verify computes before its batch check -> (status, indices or None, signing root):
    MALFORMED > NO_CACHE > NO_COMMITTEE > BITFIELD_LENGTH > UNKNOWN_VALIDATOR (an index at or beyond the pubkey table,
    ValidatorUnknown); the signing root of every well-framed record, zeros for a malformed one."""
    att = parse(ssz, electra)
    if att is None:
        return MALFORMED, None, bytes(32)
    root = signing_root(att["data"], fork_info, gvr)
    status, indices = get_attesting_indices(att, electra, caches)
    if status == OK and len(indices) and int(indices.max()) >= table_len:
        status = UNKNOWN_VALIDATOR
    return status, indices, root
