"""Merkle proofs by generalized index from resident BeaconStates (lhb200_state_proofs) and BeaconBlock bodies
(lhb200_beacon_block_body_proofs).  Every branch is checked against the from-spec proofs of tests/ssz_proof_spec.py,
and every returned root against lhb200_state_root / the spec root.  State models and chain helpers are the ones of
tests/test_state_lists_gpu.py."""
import copy
import ctypes as C
import gc
import struct

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200.synthetic import beacon_block_deneb, beacon_block_electra, beacon_state_deneb_ssz
from tests import ssz_spec
from tests.ssz_proof_spec import Prover, expand, root_from_branch
from tests.test_state_lists_gpu import StateModel, apply, deposits, header_bytes, patch, rb, resident

FORKS = ["altair", "bellatrix", "capella", "deneb", "electra"]


def top_depth(fork):
    return 6 if fork == "electra" else 5


def light_client(fork):
    from lighthouse_b200 import tree_hash as T
    if fork == "electra":
        return [T.FINALIZED_ROOT_INDEX_ELECTRA, T.CURRENT_SYNC_COMMITTEE_INDEX_ELECTRA, T.NEXT_SYNC_COMMITTEE_INDEX_ELECTRA]
    return [T.FINALIZED_ROOT_INDEX, T.CURRENT_SYNC_COMMITTEE_INDEX, T.NEXT_SYNC_COMMITTEE_INDEX]


def tree_gindices(t, v, g, rng, out, recurse=True, per_level=3):
    """Gindices inside the value v of type t whose root is node g: the length chunk of a list, and at every level of its
    chunk tree the first and last nodes, random ones, and nodes past the length; recursing into the fields of
    containers (not into list elements: the device refuses below a record root)."""
    tree, length = expand(t, v)
    base = g
    if length is not None:
        out += [2 * g, 2 * g + 1]
        base = 2 * g
    n = len(tree.chunks)
    for h in range(tree.depth):              # h levels above the leaves... down to the leaves (h = 0)
        width = 1 << (tree.depth - h)
        have = (n + (1 << h) - 1) >> h       # nodes holding data at this level
        picks = {0, max(have - 1, 0), min(have, width - 1), width - 1}
        picks |= {int(x) for x in rng.integers(0, width, size=per_level)}
        if have:
            picks |= {int(x) for x in rng.integers(0, have, size=per_level)}
        out += [(base << (tree.depth - h)) + i for i in sorted(picks)]
    if recurse and t[0] == "container":
        for k, (ft, fv) in enumerate(tree.children):
            sub = (base << tree.depth) + k
            if ft[0] == "container" or ft[0] in ("vector", "list", "bytelist") or (ft[0] == "bytes" and ft[1] > 48):
                tree_gindices(ft, fv, sub, rng, out, recurse=ft[0] == "container", per_level=per_level)


def state_gindices(model, rng, per_level=3):
    """The light-client gindices, gindex 1, every leaf of the top tree (padding included) and tree_gindices of every
    field."""
    d = top_depth(model.fork)
    value = ssz_spec.deserialize(model.typ, model.ssz())
    out = light_client(model.fork) + [1] + [(1 << d) + k for k in range(1 << d)]
    for k, (name, ft) in enumerate(model.typ[1]):
        tree_gindices(ft, value[name], (1 << d) + k, rng, out, per_level=per_level)
    return out, Prover(model.typ, value)


def check(st, model, gindices, prover, want_root=None):
    root, branches = st.proofs(gindices)
    assert root == prover.root()
    assert root == st.root()
    if want_root is not None:
        assert root == want_root
    bad = [g for g, b in zip(gindices, branches) if b != prover.proof(g)]
    assert not bad, f"{len(bad)} of {len(gindices)} branches differ, first gindices {bad[:8]}"
    return root


@pytest.mark.gpu
@pytest.mark.parametrize("fork", FORKS)
def test_staged_handles(gpu, fork):
    """Non-incremental handles of every fork: every list, vector and container is entered through the levels a proof
    rebuilds, the plan's ops or its zero operands."""
    from lighthouse_b200 import tree_hash as T
    gc.collect()
    model = StateModel(beacon_state_deneb_ssz(300, seed=11, fork=fork, n_votes=20, n_summaries=9, n_hist_roots=13,
                                              n_pending=(30, 9, 3)), fork)
    st = T.ResidentState(model.ssz(), fork)
    gis, prover = state_gindices(model, np.random.default_rng(3))
    check(st, model, gis, prover)
    assert st.compute_merkle_proof(light_client(fork)[0]) == prover.proof(light_client(fork)[0])
    assert st.proofs([1]) == (prover.root(), [[]])
    st.release()


@pytest.mark.gpu
@pytest.mark.parametrize("n_validators", [20_000, 32_760])
def test_chain_replay_proofs(gpu, n_validators):
    """A converted Deneb handle follows slots of edits and proves after each one with no explicit root first; 32 760 + 16
    deposits lifts the per-validator lists past a power of two, so paths run above their old top."""
    rng = np.random.default_rng(n_validators + 7)
    model = StateModel(beacon_state_deneb_ssz(n_validators, seed=3, n_votes=5, n_summaries=3), "deneb")
    st = resident(model)
    for slot in range(4):
        patch(st, model, 40, 0, struct.pack("<Q", 7000 + slot))
        nv = model.length("validators")
        for vi in rng.choice(nv, size=10, replace=False):
            patch(st, model, "validators", 121 * int(vi) + 80, struct.pack("<Q", int(rng.integers(1, 1 << 40))))
            patch(st, model, "balances", 8 * int(vi), struct.pack("<Q", int(rng.integers(1, 1 << 40))))
        apply(st, model, deposits(rng, model, 16))
        apply(st, model, [("eth1_data_votes", model.length("eth1_data_votes") + 1, model.length("eth1_data_votes"),
                           rb(rng, 72))])
        hdr = header_bytes(rng, "deneb", int(rng.integers(0, 33)))
        st.set_payload_header(hdr)
        model.parts["latest_execution_payload_header"][:] = hdr
        gis, prover = state_gindices(model, rng, per_level=2)
        check(st, model, gis, prover)
    st.release()


@pytest.mark.gpu
def test_converted_electra_lists(gpu):
    """The pending lists and historical_summaries of a converted Electra handle: length chunks, ladders synthesised
    above the current top, left spine nodes hashed on the device, and an emptied list."""
    rng = np.random.default_rng(5)
    model = StateModel(beacon_state_deneb_ssz(2000, seed=4, fork="electra", n_votes=3, n_summaries=5,
                                              n_pending=(40, 17, 0)), "electra")
    st = resident(model)
    apply(st, model, deposits(rng, model, 24))
    apply(st, model, [("historical_summaries", model.length("historical_summaries") + 1,
                       model.length("historical_summaries"), rb(rng, 64)),
                      ("pending_partial_withdrawals", 0, 0, b"")])
    gis, prover = state_gindices(model, rng)
    check(st, model, gis, prover)
    st.release()


@pytest.mark.gpu
def test_clones_prove_independently(gpu):
    """Two divergent clones each prove their own state; a clone proves after its source is released."""
    rng = np.random.default_rng(9)
    model = StateModel(beacon_state_deneb_ssz(3000, seed=6, n_votes=5, n_summaries=3), "deneb")
    parent = resident(model)
    apply(parent, model, [("eth1_data_votes", 6, 5, rb(rng, 72))])
    a, b = parent.clone(), parent.clone()
    ma, mb = copy.deepcopy(model), copy.deepcopy(model)
    apply(a, ma, deposits(rng, ma, 40))
    patch(b, mb, "balances", 8 * 17, struct.pack("<Q", 123456789))
    apply(b, mb, [("eth1_data_votes", 0, 0, b"")])
    for st, m in ((a, ma), (b, mb), (parent, model)):
        gis, prover = state_gindices(m, rng, per_level=2)
        check(st, m, gis, prover)
    parent.release()
    gc.collect()
    patch(a, ma, "validators", 121 * 5 + 80, struct.pack("<Q", 99))
    gis, prover = state_gindices(ma, rng, per_level=2)
    check(a, ma, gis, prover)
    a.release()
    b.release()


@pytest.mark.gpu
def test_hundred_thousand_validator_proofs(gpu):
    """One call, 100 000 validator-record proofs: a sample against hashlib, all of them through
    lhb200_verify_merkle_proofs; then the launch count of a call on a rooted incremental handle."""
    from lighthouse_b200 import _ffi
    from lighthouse_b200 import tree_hash as T
    n = 100_000
    ssz = beacon_state_deneb_ssz(n, seed=12, n_votes=4, n_summaries=2)
    model = StateModel(ssz, "deneb")
    st = T.ResidentState(ssz, "deneb")
    g0 = (2 * (32 + 11)) << 40
    gis = np.arange(n, dtype=np.uint64) + np.uint64(g0)
    root, flat = st.proofs(gis, raw=True)
    assert root == st.root()
    depth = 46
    assert flat.size == n * depth * 32
    vals = bytes(model.parts["validators"])
    leaves = T.validator_roots(vals)
    rng = np.random.default_rng(1)
    for i in rng.choice(n, size=40, replace=False).tolist():
        branch = [flat[32 * (depth * i + k): 32 * (depth * i + k + 1)].tobytes() for k in range(depth)]
        leaf = ssz_spec.hash_tree_root(S.Validator, ssz_spec.deserialize(S.Validator, vals[121 * i: 121 * i + 121]))
        assert leaves[32 * i: 32 * i + 32] == leaf
        assert root_from_branch(leaf, branch, int(gis[i])) == root
    ok = C.create_string_buffer(n)
    idx = np.arange(n, dtype=np.uint64) + np.uint64(g0 - (1 << depth))
    roots = root * n
    p_l, k1 = _ffi.buf(leaves)
    p_r, k2 = _ffi.buf(roots)
    _ffi.check(_ffi.lib.lhb200_verify_merkle_proofs(p_l, flat.ctypes.data, depth, idx.ctypes.data, p_r, n, ok),
               "lhb200_verify_merkle_proofs")
    assert ok.raw == b"\x01" * n
    st.enable_incremental()
    st.root()
    before = _ffi.lib.lhb200_launch_count()
    st.root()
    per_root = _ffi.lib.lhb200_launch_count() - before
    before = _ffi.lib.lhb200_launch_count()
    st.proofs(gis[:1000])
    assert _ffi.lib.lhb200_launch_count() - before == per_root + 1
    assert T.debug_proof_gather_ms() >= 0
    st.release()


@pytest.mark.gpu
def test_on_demand_levels_launch_count(gpu):
    """historical_roots has no resident levels: a proof into it rebuilds its ceil_log2(n) - 1 inner levels."""
    from lighthouse_b200 import _ffi
    from lighthouse_b200 import tree_hash as T
    model = StateModel(beacon_state_deneb_ssz(100, seed=2, n_hist_roots=700, n_votes=2, n_summaries=2), "deneb")
    st = T.ResidentState(model.ssz(), "deneb")
    st.root()
    before = _ffi.lib.lhb200_launch_count()
    st.root()
    per_root = _ffi.lib.lhb200_launch_count() - before
    g = ((2 * (32 + 7)) << 24) + 699
    before = _ffi.lib.lhb200_launch_count()
    root, (branch,) = st.proofs([g])
    assert _ffi.lib.lhb200_launch_count() - before == per_root + 1 + (10 - 1)
    prover = Prover(model.typ, ssz_spec.deserialize(model.typ, model.ssz()))
    assert branch == prover.proof(g) and root == prover.root()
    st.release()


@pytest.mark.gpu
def test_refusals_leave_the_handle(gpu):
    from lighthouse_b200 import _ffi
    from lighthouse_b200 import tree_hash as T
    model = StateModel(beacon_state_deneb_ssz(500, seed=8, n_votes=3, n_summaries=2), "deneb")
    st = resident(model)
    want = st.root()
    patch(st, model, "balances", 0, struct.pack("<Q", 777))    # pending: a refused call must not consume it
    bad = [0, (32 + 2) * 2,                                   # gindex 0, below the u64 slot
           ((2 * (32 + 11)) << 40) * 2,                       # below a validator root
           ((2 * (32 + 12)) << 38) * 2 + 1,                   # below a packed balances chunk
           ((((32 + 22) * 2) << 9) + 3) * 2,                  # below a sync-committee pubkey root
           ((32 + 22) * 2 + 1) * 2]                           # below the aggregate pubkey root
    for g in bad:
        with pytest.raises(_ffi.Lhb200Error) as e:
            st.proofs([105, g])
        assert e.value.code == _ffi.EINVAL
    prover = Prover(model.typ, ssz_spec.deserialize(model.typ, model.ssz()))
    root, (branch,) = st.proofs([105])
    assert root == prover.root() != want and branch == prover.proof(105)
    st.release()
    sh = T.ShardedState(beacon_state_deneb_ssz(2048, seed=1), 0, 2)
    out, r = C.create_string_buffer(32 * 8), C.create_string_buffer(32)
    g = (C.c_uint64 * 1)(105)
    assert _ffi.lib.lhb200_state_proofs(sh._h, g, 1, out, r) == _ffi.EINVAL
    sh.release()


# ---- blocks ---------------------------------------------------------------------------------------------------------
def make_block(fork, seed, **kw):
    if fork == "electra":
        return beacon_block_electra(seed=seed, n_attestations=2, n_transactions=4, **kw)
    return beacon_block_deneb(seed=seed, n_attestations=4, n_transactions=4, fork=fork, **kw)


def blind(fork, value):
    from lighthouse_b200 import synthetic
    ep = value["body"]["execution_payload"]
    pt = dict(S.EXECUTION_PAYLOAD_BY_FORK[fork][1])
    if fork == "electra":
        roots = [ssz_spec.hash_tree_root(pt[k], ep[k])
                 for k in ("transactions", "withdrawals", "deposit_requests", "withdrawal_requests")]
        return synthetic.blind_block_electra(value, *roots)
    wr = ssz_spec.hash_tree_root(pt["withdrawals"], ep["withdrawals"]) if "withdrawals" in ep else bytes(32)
    return synthetic.blind_block_deneb(value, ssz_spec.hash_tree_root(pt["transactions"], ep["transactions"]), wr, fork)


def body_gindices(fork, value, rng):
    out = list(range(16, 32)) + [1]
    body_t = S.BEACON_BLOCK_BODY_BY_FORK[fork]
    for k, (name, ft) in enumerate(body_t[1]):
        if name in ("execution_payload", "blob_kzg_commitments", "eth1_data", "sync_aggregate"):
            tree_gindices(ft, value["body"][name], 16 + k, rng, out, recurse=False)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fork", FORKS)
def test_body_proofs(gpu, fork):
    """Every body field, the payload (25) and commitments (27), every commitment against a restatement of
    verify_blob_sidecar_inclusion_proof (blob_sidecar.rs:197-221), full and blinded bodies, a batch with mixed block_of."""
    from lighthouse_b200 import tree_hash as T
    rng = np.random.default_rng(21)
    blocks = [make_block(fork, 30 + i) for i in range(3)]
    provers = [Prover(S.BEACON_BLOCK_BODY_BY_FORK[fork], v["body"]) for v, _ in blocks]
    proofs = []
    for i, (v, _) in enumerate(blocks):
        proofs += [(i, g) for g in body_gindices(fork, v, rng)]
        if fork in ("deneb", "electra"):
            proofs += [(i, T.kzg_commitment_gindex(j)) for j in range(len(v["body"]["blob_kzg_commitments"]))]
    order = rng.permutation(len(proofs))
    proofs = [proofs[j] for j in order]
    body_roots, branches = T.beacon_block_body_proofs([s for _, s in blocks], proofs, fork)
    assert body_roots == [p.root() for p in provers]
    for (b, g), br in zip(proofs, branches):
        assert br == provers[b].proof(g), (b, g)
        commitments = blocks[b][0]["body"].get("blob_kzg_commitments", [])
        if 0 <= g - 54 * 4096 < len(commitments):   # is_valid_merkle_branch(commitment root, proof, 17, index, body_root)
            leaf = ssz_spec.hash_tree_root(("bytes", 48), commitments[g - 54 * 4096])
            assert len(br) == T.KZG_COMMITMENT_INCLUSION_PROOF_DEPTH
            assert root_from_branch(leaf, br, g) == body_roots[b]
    if fork != "altair":
        blinded = [blind(fork, v) for v, _ in blocks]
        sel = [(i, g) for i in range(3) for g in (T.EXECUTION_PAYLOAD_INDEX, 16, 1) + ((27,) if fork in ("deneb", "electra") else ())]
        r_full, b_full = T.beacon_block_body_proofs([s for _, s in blocks], sel, fork)
        r_blind, b_blind = T.beacon_block_body_proofs([s for _, s in blinded], sel, fork, blinded=True)
        assert r_full == r_blind and b_full == b_blind


@pytest.mark.gpu
def test_electra_deposit_requests_and_batches(gpu):
    """An Electra block with 128 deposit requests (hashed by the record kernel: its levels are rebuilt for the proof),
    and a 32-block batch with mixed block_of."""
    from lighthouse_b200 import tree_hash as T
    v, s = beacon_block_electra(seed=77, n_attestations=1, n_transactions=2, n_deposit_requests=128)
    prover = Prover(S.BeaconBlockBodyElectra, v["body"])
    dr = ((((25 << 5) + 17) * 2) << 13)
    gis = [dr + i for i in (0, 1, 64, 127, 128, 8191)] + [dr >> 3, dr >> 7, dr // (1 << 13) + 1]
    roots, branches = T.beacon_block_body_proofs([s], [(0, g) for g in gis], "electra")
    assert roots == [prover.root()]
    assert branches == [prover.proof(g) for g in gis]
    rng = np.random.default_rng(4)
    blocks = [beacon_block_deneb(seed=100 + i, n_attestations=2, n_transactions=3) for i in range(32)]
    provers = [Prover(S.BeaconBlockBodyDeneb, b["body"]) for b, _ in blocks]
    proofs = [(int(rng.integers(0, 32)), g) for g in [25, 27, T.kzg_commitment_gindex(0), T.kzg_commitment_gindex(5),
                                                       T.kzg_commitment_gindex(6), 19, 1] * 20]
    roots, branches = T.beacon_block_body_proofs([b for _, b in blocks], proofs, "deneb")
    assert roots == [p.root() for p in provers]
    assert all(br == provers[b].proof(g) for (b, g), br in zip(proofs, branches))


@pytest.mark.gpu
def test_same_gindices_in_several_blocks(gpu):
    """One call over Electra blocks whose deposit-request lists are folded by the record kernel (65 and 200 requests,
    levels rebuilt per block) or by ops (5), proving the same element gindices in every block, interleaved: each proof
    is taken in its own block's tree, with its own block's siblings above it."""
    from lighthouse_b200 import tree_hash as T
    counts = [65, 200, 5, 200]
    blocks = [beacon_block_electra(seed=300 + i, n_attestations=1, n_transactions=2, n_deposit_requests=c)
              for i, c in enumerate(counts)]
    provers = [Prover(S.BeaconBlockBodyElectra, v["body"]) for v, _ in blocks]
    dr = ((((25 << 5) + 17) * 2) << 13)
    gis = [dr + i for i in (0, 3, 64, 66, 199, 255)] + [dr >> 2, dr >> 8, dr // (1 << 13) + 1, 25, 27]
    proofs = [(b, g) for g in gis for b in (0, 1, 2, 3)]
    proofs += [(b, g) for b in (3, 2, 1, 0) for g in gis]
    roots, branches = T.beacon_block_body_proofs([s for _, s in blocks], proofs, "electra")
    assert roots == [p.root() for p in provers]
    bad = [(b, g) for (b, g), br in zip(proofs, branches) if br != provers[b].proof(g)]
    assert not bad, bad[:8]
    for (b, g), br in zip(proofs, branches):
        assert root_from_branch(provers[b].node(g), br, g) == roots[b]


@pytest.mark.gpu
def test_body_proof_refusals(gpu):
    from lighthouse_b200 import _ffi
    from lighthouse_b200 import tree_hash as T
    v, s = make_block("deneb", 5)
    tx = ((((25 << 5) + 13) * 2) << 20)   # transactions[0] root: a byte string
    for bad in ([(0, tx * 2)], [(0, tx * 2 + 1)], [(1, 25)], [(0, 0)], [(0, T.kzg_commitment_gindex(0) * 2)]):
        with pytest.raises(_ffi.Lhb200Error) as e:
            T.beacon_block_body_proofs([s], bad, "deneb")
        assert e.value.code == _ffi.EINVAL
    with pytest.raises(_ffi.Lhb200Error) as e:
        T.beacon_block_body_proofs([s[:300]], [(0, 25)], "deneb")
    assert e.value.code == _ffi.EINVAL
    roots, (branch,) = T.beacon_block_body_proofs([s], [(0, tx)], "deneb")
    assert branch == Prover(S.BeaconBlockBodyDeneb, v["body"]).proof(tx)
