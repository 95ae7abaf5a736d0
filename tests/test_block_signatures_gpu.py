"""lhb200_block_signatures_verify against the restatement of tests/block_signature_spec.py: the verdict, block_status and
the whole sets table (kinds, items, statuses, signing roots) for Base to Electra blocks signed with the interop keys, at
2 048 to 500 000 validators, one block and 32-block segments; flipped signatures; construction codes; the gossip path;
bit-exactness with Batch.upload_indexed over the restatement's sets; launch counts; refusals; a concurrent
lhb200_attestations_verify caller.  The test without a device runs in the CPU suite."""
import threading

import numpy as np
import pytest

from lighthouse_b200 import synthetic as SY
from tests import block_signature_spec as B
from tests import committee_spec as CS

EPOCH = 100
STATE_FORK = (bytes.fromhex("03000000"), bytes.fromhex("04000000"), EPOCH - 20)
VERSIONS = (bytes.fromhex("00000000"), bytes.fromhex("02000000"))
_worlds, _keys = {}, {}


def interop_keys(n):
    if n not in _keys:
        from lighthouse_b200 import bls
        sks = SY.interop_secret_keys(n)
        pk48, pk96 = bls.sk_to_pk(b"".join(s.to_bytes(32, "big") for s in sks))
        _keys[n] = (sks, pk48, pk96)
    return _keys[n]


class World:
    """A resident state of n validators at EPOCH carrying the interop keys, its restated view, device and host committee
    caches of EPOCH - 1 and EPOCH, and a pubkey table of the first `table_len` interop keys."""

    def __init__(self, n, fork, table_len=None, sync_members=None, csc_patch=None):
        from lighthouse_b200 import bls, tree_hash as T
        self.n, self.fork = n, fork
        self.sks, pk48, pk96 = interop_keys(n)
        ssz = bytearray(SY.block_signature_state(n, fork, EPOCH * 32 + 9, STATE_FORK, pk48, sync_members))
        if csc_patch is not None:   # member 0's key replaced by a key no validator holds
            ssz[SY.O_STATE_CSC:SY.O_STATE_CSC + 48] = csc_patch
        self.ssz = bytes(ssz)
        self.state = T.ResidentState(self.ssz, fork)
        self.view = B.StateView(self.ssz, fork)
        s = CS.State(self.ssz)
        self.epochs = (EPOCH - 1, EPOCH)
        self.host = [CS.committee_cache(s, e) for e in self.epochs]
        self.dev = [self.state.device_committee_cache(e) for e in self.epochs]
        self.table_len = n if table_len is None else table_len
        self.table = bls.PubkeyTable(n)
        self.table.append(pk96[:96 * self.table_len])

    def host_cache(self, e):
        from lighthouse_b200.committees import CommitteeCache
        c = self.host[self.epochs.index(e)]
        return CommitteeCache(c["epoch"], c["shuffling"], c["positions"], c["committees_per_slot"], c["seed"])


def world(n, fork, **kw):
    key = (n, fork, tuple(sorted(kw.items())))
    if key not in _worlds:
        _worlds[key] = World(n, fork, **kw)
    return _worlds[key]


def blocks(w, n_blocks, n_atts=4, seed=0, **kw):
    """n_blocks signed blocks at consecutive slots of EPOCH, each with n_atts attestations of the previous epoch"""
    from lighthouse_b200 import tree_hash as T
    electra = w.fork == "electra"
    out, roots = [], []
    hc = w.host_cache(EPOCH - 1)
    for k in range(n_blocks):
        slot = EPOCH * 32 + k
        atts = SY.signed_attestations(hc, "electra" if electra else "aggregate", n_atts, w.sks, STATE_FORK,
                                      w.view.gvr, seed=seed + k, fill=0.9) if n_atts else []
        kw_k = dict(kw)
        proposer = kw_k.pop("proposer", w.view.proposers[slot % 32])
        kw_k.setdefault("sync_committee", w.view.sync)
        b, r = SY.signed_beacon_block(w.fork, slot, proposer, w.sks, STATE_FORK, w.view.gvr, VERSIONS,
                                      lambda m: T.beacon_block_roots([m], w.fork)[0], seed=seed + k, attestations=atts,
                                      n_validators=w.n, **kw_k)
        out.append(b)
        roots.append(r)
    return out, roots


def run(w, blks, roots, skip_proposal=False, rands=None, check=True):
    """The call, with every output checked against the restatement -> (ok, block_status, sets, spec sets)"""
    from lighthouse_b200 import block_signatures as BS
    ok, st, sets = BS.verify_block_signatures(blks, w.fork, w.state, w.dev, w.table, VERSIONS, roots, rands,
                                              skip_proposal)
    want, want_st, constructed = B.segment(blks, w.fork, w.view, w.host, w.table_len, VERSIONS, roots, skip_proposal)
    if check:
        assert [(s[0], s[1], s[2]) for s in sets] == [(x["block"], x["item"], x["kind"]) for x in want]
        assert [s[4] for s in sets] == [x["root"] for x in want]
        assert [s[3] for s in sets] == [x["status"] for x in want]
        assert st.tolist() == want_st
        if not constructed:
            assert not ok
    return ok, st, sets, want


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["base", "altair", "capella", "deneb", "electra"])
@pytest.mark.parametrize("n", [2048, 20_000, 500_000])
def test_segments_match_restatement(gpu, fork, n):
    w = world(n, fork)
    for n_blocks in (1, 32):
        blks, roots = blocks(w, n_blocks, n_atts=4 if fork != "electra" else 2)
        ok, st, sets, _ = run(w, blks, roots)
        assert ok and not st.any(), st


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["deneb", "electra"])
def test_flipped_signature_of_each_kind(gpu, fork):
    w = world(20_000, fork)
    blks, roots = blocks(w, 2)
    ok, _, sets, want = run(w, blks, roots)
    assert ok
    for j, x in enumerate(want):
        if x["block"] != 0 or x["kind"] in [y["kind"] for y in want[:j] if y["block"] == 0]:
            continue   # the first set of each kind in block 0
        sig = x["signature"]
        at = blks[0].find(sig)
        assert at >= 0
        replacement = want[-1]["signature"] if want[-1]["signature"] != sig else want[-2]["signature"]
        bad = blks[0][:at] + replacement + blks[0][at + 96:]
        ok, _, _, _ = run(w, [bad, blks[1]], roots, check=False)
        assert not ok, x["kind"]


@pytest.mark.gpu
def test_gossip_path_skips_the_proposal(gpu):
    w = world(2048, "deneb")
    blks, roots = blocks(w, 2)
    bad = blks[0][:4] + blks[1][4:100] + blks[0][100:]   # another block's proposal signature
    assert not run(w, [bad], roots[:1])[0]
    assert run(w, [bad], roots[:1], skip_proposal=True)[0]
    # a wrong block.proposer_index: INCORRECT_PROPOSER, unless the proposal is skipped (the RANDAO set takes the key
    # of the state's proposer)
    wrong = (w.view.proposers[0] + 1) % w.n
    blks, roots = blocks(w, 1)
    bad = blks[0][:108] + wrong.to_bytes(8, "little") + blks[0][116:]
    ok, st, sets, _ = run(w, [bad], roots)
    assert not ok and st[0] == B.INCORRECT_PROPOSER
    ok, st, sets, _ = run(w, [bad], roots, skip_proposal=True)
    assert ok and sets[0][2] == B.RANDAO and not st.any()


@pytest.mark.gpu
def test_construction_codes(gpu):
    # an exit index between the table length and the state's validator count: UNKNOWN_VALIDATOR
    w = world(2048, "deneb", table_len=2000)
    blks, roots = blocks(w, 1, n_atts=0, n_exits=2, n_proposer_slashings=0, n_attester_slashings=0,
                         sync_participation=0)
    body_at = 100 + int.from_bytes(blks[0][180:184], "little")
    exit_at = body_at + int.from_bytes(blks[0][body_at + 216:body_at + 220], "little")
    blks = [blks[0][:exit_at + 8] + (2010).to_bytes(8, "little") + blks[0][exit_at + 16:]]
    ok, st, sets, _ = run(w, blks, roots)
    assert not ok and B.UNKNOWN_VALIDATOR in [s[3] for s in sets]
    # a block of another epoch: SLOT_OUT_OF_BOUNDS
    w = world(2048, "deneb")
    blks, roots = blocks(w, 1)
    from lighthouse_b200 import tree_hash as T
    b2, r2 = SY.signed_beacon_block("deneb", (EPOCH + 1) * 32 + 1, 0, w.sks, STATE_FORK, w.view.gvr, VERSIONS,
                                    lambda m: T.beacon_block_roots([m], "deneb")[0], sync_committee=w.view.sync,
                                    n_validators=w.n)
    ok, st, _, _ = run(w, blks + [b2], roots + [r2])
    assert not ok and st.tolist() == [0, B.SLOT_OUT_OF_BOUNDS]
    # a sync-committee key absent from the registry
    w2 = world(2048, "altair", csc_patch=b"\xaa" * 48)
    blks, roots = blocks(w2, 2, sync_participation=1.0, sync_committee=[0] + w2.view.sync[1:])
    ok, st, _, _ = run(w2, blks, roots)
    assert not ok and st.tolist() == [B.PUBKEY_DECOMPRESSION] * 2
    # zero participation: no set with the infinity signature, a keyless set (verify status 4) with another
    blks, roots = blocks(w, 1, sync_participation=0)
    ok, st, sets, _ = run(w, blks, roots)
    assert ok and B.SYNC_AGGREGATE not in [s[2] for s in sets]
    body_at = 100 + int.from_bytes(blks[0][180:184], "little")
    bad = blks[0][:body_at + 284] + blks[0][4:100] + blks[0][body_at + 380:]
    ok, st, sets, _ = run(w, [bad], roots)
    assert not ok and [s[3] for s in sets if s[2] == B.SYNC_AGGREGATE] == [B.NO_KEYS]


def explicit_route(w, blks, roots, rands=None):
    """The restatement's sets through an explicit-key Batch.upload (96-byte keys, no pubkey table) in the call's batch
    order (the sets other than attestations, then the attestations) -> (ok, gt)"""
    from lighthouse_b200 import bls
    want = B.segment(blks, w.fork, w.view, w.host, w.table_len, VERSIONS, roots)[0]
    order = [j for j, x in enumerate(want) if x["kind"] != B.ATTESTATION] + \
            [j for j, x in enumerate(want) if x["kind"] == B.ATTESTATION]
    table96 = np.frombuffer(interop_keys(w.n)[2], dtype=np.uint8).reshape(w.n, 96)
    sigs = b"".join(want[j]["signature"] for j in order)
    msgs = b"".join(want[j]["root"] for j in order)
    pks = b"".join(B.key96(k, table96) for j in order for k in want[j]["keys"])
    offs = np.cumsum([0] + [len(want[j]["keys"]) for j in order])
    b = bls.Batch(len(order), len(pks) // 96)
    b.upload(sigs, msgs, pks, offs, None if rands is None else rands[order])
    b.enqueue()
    out = b.result(), b.gt_bytes()
    b.destroy()
    return out


@pytest.mark.gpu
def test_bit_exact_with_explicit_key_upload(gpu):
    """The same sets, BLS-to-execution changes included, through an explicit-key upload with the same scalars: the
    same verdict and final-exponentiated product."""
    from lighthouse_b200 import block_signatures as BS
    w = world(20_000, "deneb")
    blks, roots = blocks(w, 3)
    want = B.segment(blks, w.fork, w.view, w.host, w.table_len, VERSIONS, roots)[0]
    assert B.BLS_CHANGE in [x["kind"] for x in want]
    rands = np.random.default_rng(4).integers(1, 1 << 63, len(want), dtype=np.uint64)
    ok, _, _, _ = run(w, blks, roots, rands=rands)
    gt, _ = BS.last_batch_check()
    ok2, gt2 = explicit_route(w, blks, roots, rands)
    assert ok and ok2 and gt == gt2


@pytest.mark.gpu
def test_bls_change_keys_that_do_not_validate(gpu):
    """from_bls_pubkey at infinity, off the curve and outside the subgroup: PUBKEY_DECOMPRESSION on those sets"""
    w = world(2048, "capella")
    blks, roots = blocks(w, 2, n_bls_changes=3, bls_change_pubkeys=B.bad_pubkeys())
    ok, st, sets, _ = run(w, blks, roots)
    assert not ok and st.tolist() == [B.PUBKEY_DECOMPRESSION] * 2
    assert [s[3] for s in sets if s[2] == B.BLS_CHANGE] == [B.PUBKEY_DECOMPRESSION] * 6


@pytest.mark.gpu
def test_launches_and_syncs_do_not_depend_on_n_or_validators(gpu):
    """The call's own launches (the batch check's excluded) and its host synchronises are the same for 1 or 16 blocks
    and for 2 048 or 20 000 validators."""
    from lighthouse_b200 import block_signatures as BS
    counts = []
    for n, n_blocks in ((2048, 1), (2048, 16), (20_000, 4)):
        w = world(n, "deneb")
        blks, roots = blocks(w, n_blocks)
        assert run(w, blks, roots, check=False)[0]
        counts.append(BS.last_counts())
    assert counts[0] == counts[1] == counts[2], counts
    # proposer draw 4, sync resolve 1, change keys 2, roots 1, attestations 2; synchronises: 2 front, 1 read-back, 1 verdict
    assert counts[0] == (10, 4), counts


@pytest.mark.gpu
def test_refusals_and_concurrent_attestation_caller(gpu):
    from lighthouse_b200 import attestations as AT, block_signatures as BS
    from lighthouse_b200._ffi import Lhb200Error, EINVAL
    w = world(2048, "deneb")
    blks, roots = blocks(w, 2)
    for bad_call in (
        lambda: BS.verify_block_signatures([], "deneb", w.state, w.dev, w.table, VERSIONS, []),
        lambda: BS.verify_block_signatures(blks, "capella", w.state, w.dev, w.table, VERSIONS, roots),
        lambda: BS.verify_block_signatures([blks[0][:50]], "deneb", w.state, w.dev, w.table, VERSIONS, roots[:1]),
        lambda: BS.verify_block_signatures(blks, "deneb", w.state, [], w.table, VERSIONS, roots),
        lambda: BS.verify_block_signatures(blks, "deneb", w.state, w.dev, w.table, VERSIONS, roots, rands=[1]),
        lambda: BS.verify_block_signatures(blks, "deneb", w.state, w.dev, w.table, VERSIONS, roots, rands=[0] * 400),
    ):
        with pytest.raises(Lhb200Error) as e:
            bad_call()
        assert e.value.code == EINVAL
    # a body whose bls_to_execution_changes list is not a whole number of records
    body_at = 100 + int.from_bytes(blks[0][180:184], "little")
    at = body_at + 384
    o = int.from_bytes(blks[0][at:at + 4], "little")
    bad = blks[0][:at] + (o + 1).to_bytes(4, "little") + blks[0][at + 4:]
    with pytest.raises(Lhb200Error) as e:
        BS.verify_block_signatures([bad], "deneb", w.state, w.dev, w.table, VERSIONS, roots[:1])
    assert e.value.code == EINVAL
    # a concurrent attestation caller on another thread
    atts = SY.signed_attestations(w.host_cache(EPOCH), "aggregate", 16, w.sks, STATE_FORK, w.view.gvr)
    res = []

    def other():
        for _ in range(3):
            res.append(AT.verify_attestations(atts, "deneb", w.dev, w.table, STATE_FORK, w.view.gvr)[0])

    t = threading.Thread(target=other)
    t.start()
    for _ in range(3):
        assert run(w, blks, roots)[0]
    t.join()
    assert res == [True] * 3


def test_enodev_without_a_device():
    """Without lhb200_init the call refuses with ENODEV (no CPU fallback)."""
    import lighthouse_b200._ffi as F
    if F._inited is not None:
        pytest.skip("the library is initialised in this process")
    from lighthouse_b200 import block_signatures as BS  # noqa: F401
    import ctypes as C
    rc = F.lib.lhb200_block_signatures_verify(None, None, 0, 4, 0, None, None, None, 0, None, None, None, 0, None,
                                              None, None, 0, C.byref(C.c_uint64()))
    assert rc == F.ENODEV
