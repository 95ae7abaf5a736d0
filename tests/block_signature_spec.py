"""From-spec restatement of BlockSignatureVerifier::include_all_signatures (block_signature_verifier.rs:150-173) and the
sets of signature_sets.rs over a BeaconState's SSZ (no GPU): the blocks are decoded with the generic SSZ decoder of
tests/ssz_spec.py over ssz_schema, attestations are indexed by tests/attestation_spec.py, proposers come from
tests/committee_spec.py, and every set carries the status lhb200_block_signatures_verify reports before its batch check.
hashlib and numpy, and the big-integer oracle's G1 decoding (oracle/bls_ref.py) for the BLS-to-execution changes' keys.
A set's keys are validator indices, or for a change the 48-byte from_bls_pubkey itself."""
import struct

import numpy as np

from lighthouse_b200 import ssz_schema as S
from tests import attestation_spec as A
from tests import committee_spec as CS
from tests import ssz_spec

PROPOSAL, RANDAO, PROPOSER_SLASHING, ATTESTER_SLASHING, ATTESTATION, EXIT, SYNC_AGGREGATE, BLS_CHANGE, CONSOLIDATION = \
    range(9)
INCORRECT_PROPOSER, SLOT_OUT_OF_BOUNDS, PUBKEY_DECOMPRESSION = 15, 16, 17
UNKNOWN_VALIDATOR, NO_KEYS = 14, 4
DOMAIN_PROPOSER, DOMAIN_ATTESTER, DOMAIN_RANDAO, DOMAIN_EXIT, DOMAIN_SYNC = 0, 1, 2, 4, 7
DOMAIN_BLS_TO_EXECUTION_CHANGE, DOMAIN_CONSOLIDATION = 0x0A, 0x0B
O_GVR, O_FORK, O_CSC = 8, 48, 2687381
INFINITY = b"\xc0" + bytes(95)
SigningData = S.C(("object_root", S.B32), ("domain", S.B32))


def signed_block_type(fork):
    return S.C(("message", S.BEACON_BLOCK_BY_FORK[fork]), ("signature", S.B96))


def signing_root(object_root, domain):
    return A.sha(object_root + domain)


class StateView:
    """What the block sets read from a state: the slot, fork, genesis_validators_root, proposers, pubkeys and the
    current sync committee resolved to validator indices (smallest index per key)."""

    def __init__(self, ssz, fork):
        s = CS.State(ssz)
        self.slot, self.n = s.slot, len(s.validators)
        self.prev, self.cur = bytes(ssz[O_FORK:O_FORK + 4]), bytes(ssz[O_FORK + 4:O_FORK + 8])
        self.fork_epoch = struct.unpack_from("<Q", ssz, O_FORK + 8)[0]
        self.gvr = bytes(ssz[O_GVR:O_GVR + 32])
        self.proposers = CS.beacon_proposer_indices(s)
        self.sync = None
        if fork != "base":
            first = {}
            raw = np.ascontiguousarray(s.validators[:, :48]).tobytes()
            for i in range(self.n):
                first.setdefault(raw[48 * i:48 * i + 48], i)
            csc = bytes(ssz[O_CSC:O_CSC + 512 * 48])
            self.sync = [first.get(csc[48 * m:48 * m + 48]) for m in range(512)]

    def domain(self, dtype, epoch):
        return A.compute_domain(dtype, self.prev if epoch < self.fork_epoch else self.cur, self.gvr)


def key_validate(pk48):
    """PublicKey::deserialize + key_validate: the uncompressed 96-byte key, or None for an infinity, undecodable,
    off-curve or non-subgroup key"""
    from oracle import bls_ref as R
    try:
        p = R.g1_decompress(bytes(pk48))
    except ValueError:
        return None
    if p is None or not R.g1_in_subgroup(p):
        return None
    return R.g1_uncompressed(p)


def bad_pubkeys():
    """Compressed G1 encodings key_validate refuses: (infinity, off the curve, on the curve outside the subgroup)"""
    from oracle import bls_ref as R
    off = nonsub = None
    x = 1
    while off is None or nonsub is None:
        enc = (x | (1 << 383)).to_bytes(48, "big")   # the compression flag
        if pow((x ** 3 + 4) % R.P, (R.P - 1) // 2, R.P) != 1:
            off = off or enc
        elif nonsub is None and not R.g1_in_subgroup(R.g1_decompress(enc)):
            nonsub = enc
        x += 1
    return b"\xc0" + bytes(47), off, nonsub


def key96(k, table96):
    """A set's key as 96 uncompressed bytes: a validator index into table96, or a change's from_bls_pubkey"""
    return key_validate(k) if isinstance(k, bytes) else bytes(table96[k])


def header_root(h):
    return ssz_spec.hash_tree_root(S.BeaconBlockHeader, h)


def block_sets(signed_ssz, fork, view, caches, table_len, versions, block_root, skip_proposal=False):
    """-> the sets of one SignedBeaconBlock in push order, each a dict(kind, item, status, root, keys, signature):
    status 0 (constructed), NO_KEYS for a constructed set without keys (its verify status), or a construction code."""
    blk = ssz_spec.deserialize(signed_block_type(fork), signed_ssz)["message"]
    body, slot = blk["body"], blk["slot"]
    epoch, electra = slot // 32, fork == "electra"
    limit = min(table_len, view.n)
    out = []

    def push(kind, item, root, keys, sig, status=0):
        if status == 0 and keys is not None and any(not isinstance(k, bytes) and k >= limit for k in keys):
            status = UNKNOWN_VALIDATOR
        if status == 0 and keys is not None and not keys:
            status = NO_KEYS
        out.append({"kind": kind, "item": item, "status": status, "root": root,
                    "keys": list(keys) if status in (0, NO_KEYS) else None, "signature": sig})

    proposer = view.proposers[slot % 32]
    in_epoch = epoch == view.slot // 32
    if not skip_proposal:
        st = SLOT_OUT_OF_BOUNDS if not in_epoch else INCORRECT_PROPOSER if proposer != blk["proposer_index"] else 0
        push(PROPOSAL, 0, signing_root(block_root, view.domain(DOMAIN_PROPOSER, epoch)), [proposer],
             signed_ssz[4:100], st)
    push(RANDAO, 0, signing_root(epoch.to_bytes(8, "little") + bytes(24), view.domain(DOMAIN_RANDAO, epoch)),
         [proposer], body["randao_reveal"], 0 if in_epoch else SLOT_OUT_OF_BOUNDS)
    for j, ps in enumerate(body["proposer_slashings"]):
        for k in (0, 1):
            h = ps["signed_header_%d" % (k + 1)]
            push(PROPOSER_SLASHING, 2 * j + k,
                 signing_root(header_root(h["message"]), view.domain(DOMAIN_PROPOSER, h["message"]["slot"] // 32)),
                 [h["message"]["proposer_index"]], h["signature"])
    for j, sl in enumerate(body["attester_slashings"]):
        for k in (0, 1):
            ia = sl["attestation_%d" % (k + 1)]
            data = ssz_spec.hash_tree_root(S.AttestationData, ia["data"])
            push(ATTESTER_SLASHING, 2 * j + k,
                 signing_root(data, view.domain(DOMAIN_ATTESTER, ia["data"]["target"]["epoch"])),
                 ia["attesting_indices"], ia["signature"])
    fork_info = (view.prev, view.cur, view.fork_epoch)
    att_t = S.AttestationData
    for j, a in enumerate(body["attestations"]):
        data = S.serialize(att_t, a["data"])
        cb = sum(1 << k for k, b in enumerate(a["committee_bits"]) if b) if electra else None
        from lighthouse_b200.synthetic import attestation_ssz
        rec = attestation_ssz(np.array(a["aggregation_bits"], dtype=np.uint8), data, a["signature"], cb)
        st, idx, root = A.index_attestation(rec, electra, caches, limit, fork_info, view.gvr)
        keys = idx.tolist() if st == A.OK else None
        out.append({"kind": ATTESTATION, "item": j, "status": (NO_KEYS if st == A.OK and not keys else st),
                    "root": root, "keys": keys, "signature": a["signature"]})
    for j, ex in enumerate(body["voluntary_exits"]):
        m = ex["message"]
        d = A.compute_domain(DOMAIN_EXIT, versions[1], view.gvr) if fork in ("deneb", "electra") else \
            view.domain(DOMAIN_EXIT, m["epoch"])
        push(EXIT, j, signing_root(ssz_spec.hash_tree_root(S.VoluntaryExit, m), d), [m["validator_index"]],
             ex["signature"])
    if fork != "base":
        sa = body["sync_aggregate"]
        bits, sig = sa["sync_committee_bits"], sa["sync_committee_signature"]
        if any(bits) or sig != INFINITY:
            prev_slot = max(slot, 1) - 1
            root = signing_root(blk["parent_root"], view.domain(DOMAIN_SYNC, prev_slot // 32))
            keys = [view.sync[m] for m in range(512) if bits[m]]
            if any(k is None or k >= table_len for k in keys):
                push(SYNC_AGGREGATE, 0, root, None, sig, PUBKEY_DECOMPRESSION)
            else:
                push(SYNC_AGGREGATE, 0, root, keys, sig)
    for j, ch in enumerate(body.get("bls_to_execution_changes", [])):
        m = ch["message"]
        root = signing_root(ssz_spec.hash_tree_root(S.BlsToExecutionChange, m),
                            A.compute_domain(DOMAIN_BLS_TO_EXECUTION_CHANGE, versions[0], view.gvr))
        pk = bytes(m["from_bls_pubkey"])
        push(BLS_CHANGE, j, root, [pk], ch["signature"], 0 if key_validate(pk) else PUBKEY_DECOMPRESSION)
    if electra:
        for j, c in enumerate(body["consolidations"]):
            m = c["message"]
            push(CONSOLIDATION, j,
                 signing_root(ssz_spec.hash_tree_root(S.Consolidation, m),
                              A.compute_domain(DOMAIN_CONSOLIDATION, versions[0], view.gvr)),
                 [m["source_index"], m["target_index"]], c["signature"])
    return out


def segment(blocks, fork, view, caches, table_len, versions, block_roots, skip_proposal=False):
    """-> (sets of every block, each with its "block"; block_status list; constructed: every set built)."""
    sets, status = [], []
    for i, (b, r) in enumerate(zip(blocks, block_roots)):
        bs = block_sets(b, fork, view, caches, table_len, versions, r, skip_proposal)
        for s in bs:
            s["block"] = i
        sets += bs
        status.append(next((s["status"] for s in bs if s["status"]), 0))
    return sets, status, all(s["status"] in (0, NO_KEYS) for s in sets) and not any(
        s["status"] == NO_KEYS for s in sets)
