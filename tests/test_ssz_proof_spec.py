"""CPU-only: the from-spec Merkle proofs of tests/ssz_proof_spec.py verify against ssz_spec.hash_tree_root on small
states and block bodies of every fork, and for Altair to Deneb the light-client gindices 105 / 54 / 55 give the
branches Lighthouse builds (BeaconState::compute_merkle_proof, beacon_state.rs:2483-2557: a depth-5 MerkleTree of the
field roots, plus the finalized epoch chunk for 105).  The proof entry points refuse with ENODEV without a device."""
import ctypes as C

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200.synthetic import beacon_block_deneb, beacon_block_electra, beacon_state_deneb_ssz
from tests import merkle_tree_spec as M
from tests import ssz_spec
from tests.ssz_proof_spec import Prover, root_from_branch

FORKS = ["altair", "bellatrix", "capella", "deneb", "electra"]


def random_gindices(prover, rng, n, max_depth=64):
    """n gindices reached by random descents from the root, each stopped at a random depth or at a leaf."""
    out = []
    while len(out) < n:
        g, stop = 1, int(rng.integers(1, max_depth))
        for _ in range(stop):
            nxt = 2 * g + int(rng.integers(0, 2))
            try:
                prover.proof(nxt)
            except ValueError:
                break
            g = nxt
        out.append(g)
    return out


def check_verifies(prover, gindices):
    root = prover.root()
    for g in gindices:
        branch = prover.proof(g)
        assert len(branch) == g.bit_length() - 1
        assert root_from_branch(prover.node(g), branch, g) == root, g


@pytest.mark.parametrize("fork", FORKS)
def test_state_proofs_verify(fork):
    typ = S.BEACON_STATE_BY_FORK[fork]
    value = ssz_spec.deserialize(typ, beacon_state_deneb_ssz(40, seed=5, fork=fork, n_votes=12, n_summaries=3,
                                                             n_hist_roots=9))
    p = Prover(typ, value)
    rng = np.random.default_rng(1)
    n_fields = len(typ[1])
    top = (n_fields - 1).bit_length()
    check_verifies(p, [1] + [(1 << top) + k for k in range(1 << top)] + random_gindices(p, rng, 150))
    with pytest.raises(ValueError):
        p.proof(((1 << top) + 2) * 2)       # below the u64 slot
    with pytest.raises(ValueError):
        p.proof(0)


@pytest.mark.parametrize("fork", FORKS)
def test_body_proofs_verify(fork):
    if fork == "electra":
        value, _ = beacon_block_electra(seed=9, n_attestations=2, n_transactions=3, n_deposit_requests=3)
    else:
        value, _ = beacon_block_deneb(seed=9, n_attestations=3, n_transactions=3, fork=fork)
    typ = S.BEACON_BLOCK_BODY_BY_FORK[fork]
    p = Prover(typ, value["body"])
    rng = np.random.default_rng(2)
    check_verifies(p, [1] + list(range(16, 32)) + random_gindices(p, rng, 150))
    if fork in ("deneb", "electra"):
        from lighthouse_b200.tree_hash import kzg_commitment_gindex
        for i in range(len(value["body"]["blob_kzg_commitments"])):
            g = kzg_commitment_gindex(i)
            assert g.bit_length() - 1 == 17
            assert p.node(g) == ssz_spec.hash_tree_root(("bytes", 48), value["body"]["blob_kzg_commitments"][i])
        check_verifies(p, [27, kzg_commitment_gindex(4095)])


@pytest.mark.parametrize("fork", ["altair", "bellatrix", "capella", "deneb"])
def test_light_client_gindices_match_lighthouse(fork):
    from lighthouse_b200 import tree_hash as T
    typ = S.BEACON_STATE_BY_FORK[fork]
    value = ssz_spec.deserialize(typ, beacon_state_deneb_ssz(30, seed=8, fork=fork, n_votes=4, n_hist_roots=2))
    p = Prover(typ, value)
    leaves = [ssz_spec.hash_tree_root(ft, value[name]) for name, ft in typ[1]]
    tree = M.create(leaves, 5)
    for g, field in ((T.CURRENT_SYNC_COMMITTEE_INDEX, 22), (T.NEXT_SYNC_COMMITTEE_INDEX, 23)):
        assert p.proof(g) == M.generate_proof(tree, field, 5)[1]
    epoch = value["finalized_checkpoint"]["epoch"].to_bytes(32, "little")
    assert p.proof(T.FINALIZED_ROOT_INDEX) == [epoch] + M.generate_proof(tree, 20, 5)[1]


def test_electra_light_client_gindices():
    """Electra's 37 fields take a 64-leaf top tree: the same fields sit one level deeper."""
    from lighthouse_b200 import tree_hash as T
    typ = S.BEACON_STATE_BY_FORK["electra"]
    names = [n for n, _ in typ[1]]
    assert T.FINALIZED_ROOT_INDEX_ELECTRA == (64 + names.index("finalized_checkpoint")) * 2 + 1
    assert T.CURRENT_SYNC_COMMITTEE_INDEX_ELECTRA == 64 + names.index("current_sync_committee")
    assert T.NEXT_SYNC_COMMITTEE_INDEX_ELECTRA == 64 + names.index("next_sync_committee")
    body = [n for n, _ in S.BEACON_BLOCK_BODY_BY_FORK["electra"][1]]
    assert T.EXECUTION_PAYLOAD_INDEX == 16 + body.index("execution_payload")
    assert T.BLOB_KZG_COMMITMENTS_INDEX == 16 + body.index("blob_kzg_commitments")


def test_proof_entry_points_need_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    g = (C.c_uint64 * 1)(105)
    out, root = C.create_string_buffer(32 * 8), C.create_string_buffer(32)
    assert _ffi.lib.lhb200_state_proofs(None, g, 1, out, root) == _ffi.ENODEV
    offs = (C.c_uint64 * 2)(0, 0)
    blk = (C.c_uint32 * 1)(0)
    assert _ffi.lib.lhb200_beacon_block_body_proofs(None, offs, 1, 4, 0, blk, g, 1, out, root) == _ffi.ENODEV
    assert _ffi.lib.lhb200_debug_proof_gather_ms() < 0
