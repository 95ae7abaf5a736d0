"""CPU-only: the phase0 (Base) schema against real data.  The mainnet and Sepolia genesis states, put back together
from their golden pieces, give their golden state roots under the from-spec merkleization of tests/ssz_spec.py, and
the mainnet genesis block follows from its state root; the Base fixed sizes are the ones the device layouts assume;
the new entry point refuses with ENODEV without a device."""
import ctypes as C
import json
import os

import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic
from tests import ssz_spec
from tests.phase0_state import GOLDEN, genesis_block, genesis_state


@pytest.mark.parametrize("net", ["mainnet", "sepolia"])
def test_genesis_states_give_their_golden_roots(net):
    ssz, meta = genesis_state(net)
    value = ssz_spec.deserialize(S.BeaconStateBase, ssz)
    assert S.serialize(S.BeaconStateBase, value) == ssz
    assert ssz_spec.hash_tree_root(S.BeaconStateBase, value).hex() == meta["state_root"]
    # the one list pinned before: genesis_validators_root, which the state carries at bytes 8..40
    assert ssz_spec.hash_tree_root(S.BeaconStateBase[1][11][1], value["validators"]) == ssz[8:40]


def test_mainnet_genesis_block_root_follows_from_the_state_root():
    meta = json.load(open(os.path.join(GOLDEN, "genesis_states.json")))["mainnet"]
    assert meta["state_root"] == "7e76880eb67bbdc86250aa578958e9d0675e64e714337855204fb5abaaf82c2b"
    block = genesis_block(bytes.fromhex(meta["state_root"]))
    root = ssz_spec.hash_tree_root(S.BeaconBlockBase, block)
    assert root.hex() == meta["genesis_block_root"] == \
        "4d611d5b93fdab69013a7f0a2f961caca0c853f87cfe9595fe50038163079360"


def test_base_fixed_sizes():
    assert S.fixed_size(S.BeaconStateBase) == synthetic.BASE_FIXED == 2687377
    assert S.fixed_size(S.BeaconBlockBodyBase) == 220
    assert S.fixed_size(S.PendingAttestation) == 148
    assert len(S.BeaconStateBase[1]) == 21 and len(S.BeaconBlockBodyBase[1]) == 8
    assert "base" not in S.BLINDED_BEACON_BLOCK_BY_FORK


def test_synthetic_base_state_is_valid_ssz():
    import numpy as np
    ssz = synthetic.beacon_state_deneb_ssz(8, seed=5, fork="base", n_pending_attestations=(6, 1))
    value = ssz_spec.deserialize(S.BeaconStateBase, ssz)
    assert S.serialize(S.BeaconStateBase, value) == ssz
    lens = [len(a["aggregation_bits"]) for a in value["previous_epoch_attestations"]]
    assert lens == list(synthetic.PENDING_BIT_LENGTHS) and len(value["current_epoch_attestations"]) == 1
    rec = synthetic.pending_attestation_ssz(np.random.default_rng(1), 9, slot=77)
    assert ssz_spec.deserialize(S.PendingAttestation, rec)["data"]["slot"] == 77
    _, blk = synthetic.beacon_block_deneb(seed=4, fork="base", n_attestations=3)
    assert S.serialize(S.BeaconBlockBase, ssz_spec.deserialize(S.BeaconBlockBase, blk)) == blk


def test_set_pending_attestations_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    assert _ffi.lib.lhb200_state_set_pending_attestations(None, 15, None, 0) == _ffi.ENODEV
    n = C.c_uint64(0)
    assert _ffi.lib.lhb200_state_list_len(None, 15, C.byref(n)) == _ffi.ENODEV
