"""The block-signature restatement of tests/block_signature_spec.py pinned without a GPU: the object roots the signed
blocks are signed over against the generic merkleization of tests/ssz_spec.py, the domain rules (EIP-7044 from Deneb,
genesis-version consolidations, the sync aggregate's previous slot), push order, the construction codes, and every set
of synthetic signed blocks verifying under the C oracle."""
import struct

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic as SY
from tests import block_signature_spec as B
from tests import ssz_spec

N = 64
SLOT = 100 * 32 + 5
STATE_FORK = (bytes.fromhex("03000000"), bytes.fromhex("04000000"), 90)
VERSIONS = (bytes.fromhex("00000000"), bytes.fromhex("02000000"))
_keys = {}


def keys(oracle):
    if not _keys:
        sks = SY.interop_secret_keys(N)
        pk96 = [oracle.bls_sk_to_pk(s.to_bytes(32, "big")) for s in sks]
        _keys.update(sks=sks, pk96=pk96, pk48=b"".join(SY.g1_compress(p) for p in pk96))
    return _keys


def oracle_sign(oracle):
    def sign(sks, msgs):
        return b"".join(oracle.bls_sign(sks[32 * k:32 * k + 32], msgs[32 * k:32 * k + 32]) for k in range(len(sks) // 32))
    return sign


def block_root_fn(fork):
    return lambda msg: ssz_spec.hash_tree_root(S.BEACON_BLOCK_BY_FORK[fork], ssz_spec.deserialize(S.BEACON_BLOCK_BY_FORK[fork], msg))


def oracle_pk(oracle):
    def pk(sks):
        return b"".join(SY.g1_compress(oracle.bls_sk_to_pk(sks[32 * k:32 * k + 32])) for k in range(len(sks) // 32))
    return pk


def make(oracle, fork, slot=SLOT, **kw):
    k = keys(oracle)
    state = SY.block_signature_state(N, fork, SLOT, STATE_FORK, k["pk48"])
    view = B.StateView(state, fork)
    proposer = kw.pop("proposer", view.proposers[slot % 32])
    blk, root = SY.signed_beacon_block(fork, slot, proposer, k["sks"], STATE_FORK, view.gvr, VERSIONS,
                                       block_root_fn(fork), oracle_sign(oracle), sync_committee=view.sync, seed=3,
                                       n_validators=N, pk_fn=oracle_pk(oracle), **kw)
    return blk, root, view


def test_object_roots_against_generic_merkleization():
    rng = np.random.default_rng(1)
    h = {"slot": 7, "proposer_index": 9, "parent_root": rng.bytes(32), "state_root": rng.bytes(32), "body_root": rng.bytes(32)}
    assert SY.header_root(*h.values()) == ssz_spec.hash_tree_root(S.BeaconBlockHeader, h)
    d = SY.compute_domain(7, b"\1\2\3\4", rng.bytes(32))
    sd = {"object_root": rng.bytes(32), "domain": d}
    assert B.signing_root(sd["object_root"], d) == ssz_spec.hash_tree_root(B.SigningData, sd)
    c = {"source_index": 3, "target_index": 5, "epoch": 11}
    got = SY._sha(SY._sha(SY._chunk(3) + SY._chunk(5)) + SY._sha(SY._chunk(11) + bytes(32)))
    assert got == ssz_spec.hash_tree_root(S.Consolidation, c)
    ex = {"epoch": 4, "validator_index": 8}
    assert SY._sha(SY._chunk(4) + SY._chunk(8)) == ssz_spec.hash_tree_root(S.VoluntaryExit, ex)


@pytest.mark.parametrize("fork", ["base", "altair", "capella", "deneb", "electra"])
def test_synthetic_block_verifies_under_oracle_in_push_order(oracle, fork):
    blk, root, view = make(oracle, fork)
    sets, status, constructed = B.segment([blk], fork, view, [], N, VERSIONS, [root])
    kinds = [s["kind"] for s in sets]
    want = [B.PROPOSAL, B.RANDAO] + [B.PROPOSER_SLASHING] * 2 + [B.ATTESTER_SLASHING] * 2 + [B.EXIT] * 2
    want += [B.SYNC_AGGREGATE] if fork != "base" else []
    want += [B.BLS_CHANGE] * 2 if fork in ("capella", "deneb", "electra") else []
    want += [B.CONSOLIDATION] if fork == "electra" else []
    assert kinds == want and status == [0] and constructed
    assert [s["item"] for s in sets[2:6]] == [0, 1, 0, 1]
    k = keys(oracle)
    pks = b"".join(B.key96(v, k["pk96"]) for s in sets for v in s["keys"])
    offs = np.cumsum([0] + [len(s["keys"]) for s in sets])
    sigs, msgs = b"".join(s["signature"] for s in sets), b"".join(s["root"] for s in sets)
    ok, st = oracle.bls_verify_signature_sets(sigs, msgs, pks, offs, list(range(1, len(sets) + 1)), want_status=True)
    assert ok and not st.any()
    # the other fork's exit domain does not verify: EIP-7044 switches at Deneb
    if fork in ("capella", "deneb"):
        ex = [s for s in sets if s["kind"] == B.EXIT][0]
        d_capella = SY.compute_domain(4, VERSIONS[1], view.gvr)
        m = ssz_spec.deserialize(B.signed_block_type(fork), blk)["message"]["body"]["voluntary_exits"][0]["message"]
        assert d_capella != view.domain(4, m["epoch"])
        r = ssz_spec.hash_tree_root(S.VoluntaryExit, m)
        assert ex["root"] == B.signing_root(r, d_capella if fork == "deneb" else view.domain(4, m["epoch"]))


def exit_index_at(blk):
    """offset in the SignedBeaconBlock of the first exit's validator_index"""
    body_at = 100 + struct.unpack_from("<I", blk, 100 + 80)[0]
    return body_at + struct.unpack_from("<I", blk, body_at + 216)[0] + 8


def test_construction_codes(oracle):
    fork = "deneb"
    # a wrong block.proposer_index: INCORRECT_PROPOSER on the proposal only, nothing with skip_proposal
    blk, root, view = make(oracle, fork)
    wrong = (view.proposers[SLOT % 32] + 1) % N
    bad = blk[:108] + struct.pack("<Q", wrong) + blk[116:]
    sets, status, _ = B.segment([bad], fork, view, [], N, VERSIONS, [root])
    assert status == [B.INCORRECT_PROPOSER] and sets[0]["status"] == B.INCORRECT_PROPOSER
    sets, status, _ = B.segment([bad], fork, view, [], N, VERSIONS, [root], skip_proposal=True)
    assert status == [0] and not any(s["status"] for s in sets)
    # a block outside the state's epoch: SLOT_OUT_OF_BOUNDS on proposal and randao
    blk2, root2, _ = make(oracle, fork, slot=SLOT + 32, proposer=0)
    sets, status, _ = B.segment([blk2], fork, view, [], N, VERSIONS, [root2])
    assert [s["status"] for s in sets[:2]] == [B.SLOT_OUT_OF_BOUNDS] * 2 and status == [B.SLOT_OUT_OF_BOUNDS]
    # an exit index at the table's length: UNKNOWN_VALIDATOR on that exit
    at = exit_index_at(blk)
    bad = blk[:at] + struct.pack("<Q", N - 1) + blk[at + 8:]
    sets, status, _ = B.segment([bad], fork, view, [], N - 1, VERSIONS, [root])
    ex = [s for s in sets if s["kind"] == B.EXIT][0]
    assert ex["status"] == B.UNKNOWN_VALIDATOR and status == [B.UNKNOWN_VALIDATOR]
    # a sync-committee key no record holds, on a participating bit: PUBKEY_DECOMPRESSION
    blk, root, view = make(oracle, fork, sync_participation=1.0)
    view.sync = [None] + view.sync[1:]
    sets, status, _ = B.segment([blk], fork, view, [], N, VERSIONS, [root])
    assert [s["status"] for s in sets if s["kind"] == B.SYNC_AGGREGATE] == [B.PUBKEY_DECOMPRESSION]
    # from_bls_pubkey at infinity, off the curve, outside the subgroup: PUBKEY_DECOMPRESSION
    blk, root, view = make(oracle, fork, n_bls_changes=3, bls_change_pubkeys=B.bad_pubkeys())
    sets, status, _ = B.segment([blk], fork, view, [], N, VERSIONS, [root])
    assert [s["status"] for s in sets if s["kind"] == B.BLS_CHANGE] == [B.PUBKEY_DECOMPRESSION] * 3


def test_sync_aggregate_zero_participation_and_previous_slot(oracle):
    fork = "altair"
    blk, root, view = make(oracle, fork, sync_participation=0)
    sets, _, ok = B.segment([blk], fork, view, [], N, VERSIONS, [root])
    assert B.SYNC_AGGREGATE not in [s["kind"] for s in sets] and ok   # zero bits, infinity signature: no set
    # zero bits with another signature: a set without keys
    body_at = 100 + struct.unpack_from("<I", blk, 100 + 80)[0]
    bad = bytearray(blk)
    bad[body_at + 284:body_at + 380] = blk[4:100]
    sets, status, ok = B.segment([bytes(bad)], fork, view, [], N, VERSIONS, [root])
    assert sets[-1]["kind"] == B.SYNC_AGGREGATE and sets[-1]["status"] == B.NO_KEYS and not ok
    # the previous slot's epoch: at the fork epoch's first slot the sync set takes the previous fork's version
    blk, root, view = make(oracle, fork, slot=90 * 32, proposer=0)
    sync = [s for s in B.block_sets(blk, fork, view, [], N, VERSIONS, root) if s["kind"] == B.SYNC_AGGREGATE][0]
    parent = ssz_spec.deserialize(B.signed_block_type(fork), blk)["message"]["parent_root"]
    assert sync["root"] == B.signing_root(parent, SY.compute_domain(7, STATE_FORK[0], view.gvr))
    blk, root, view = make(oracle, fork, slot=0, proposer=0)
    sync = [s for s in B.block_sets(blk, fork, view, [], N, VERSIONS, root) if s["kind"] == B.SYNC_AGGREGATE][0]
    parent = ssz_spec.deserialize(B.signed_block_type(fork), blk)["message"]["parent_root"]
    assert sync["root"] == B.signing_root(parent, SY.compute_domain(7, STATE_FORK[0], view.gvr))
