"""The attestation restatement of tests/attestation_spec.py pinned without a GPU: its AttestationData root against the
generic merkleization of tests/ssz_spec.py over ssz_schema.AttestationData, its domain against the same merkleization of
ForkData,
one hand-built case per status in the reference's order, and the mainnet genesis state, where the single-bit
attestations of every committee of epoch 0 name every active validator exactly once."""
import struct

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic as SY
from lighthouse_b200.committees import CommitteeCache
from lighthouse_b200.synthetic import attestation_data_ssz, attestation_ssz, beacon_state_deneb_ssz
from tests import attestation_spec as A
from tests import committee_spec as CS
from tests import ssz_spec
from tests.phase0_state import genesis_state

FORK = (bytes.fromhex("03000000"), bytes.fromhex("04000000"), 10)
GVR = bytes(range(32))


def random_data(rng, slot=None, index=None, target_epoch=None):
    r = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    slot = int(rng.integers(0, 1 << 40)) if slot is None else slot
    index = int(rng.integers(0, 64)) if index is None else index
    te = int(rng.integers(0, 1 << 40)) if target_epoch is None else target_epoch
    return attestation_data_ssz(slot, index, r(), (int(rng.integers(0, 1 << 40)), r()), (te, r()))


def test_data_root_matches_generic_merkleization():
    rng = np.random.default_rng(1)
    for _ in range(20):
        data = random_data(rng)
        want = ssz_spec.hash_tree_root(S.AttestationData, ssz_spec.deserialize(S.AttestationData, data))
        assert A.attestation_data_root(data) == want == SY.attestation_data_root(data)


def test_domain_and_signing_root():
    """compute_domain = le32(type) || hash_tree_root(ForkData)[:28], the ForkData root from the generic merkleization
    (tree_hash.compute_domain hashes on the device: tests/test_attestations_gpu.py pins it)."""
    fork_data = S.C(("current_version", ("bytes", 4)), ("genesis_validators_root", S.B32))
    rng = np.random.default_rng(2)
    for _ in range(5):
        v, g = rng.integers(0, 256, 4, dtype=np.uint8).tobytes(), rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
        root = ssz_spec.hash_tree_root(fork_data, {"current_version": v, "genesis_validators_root": g})
        assert A.compute_domain(1, v, g) == b"\x01\0\0\0" + root[:28] == SY.attester_domain(v, g)
    prev, cur, fork_epoch = FORK
    for te, version in ((fork_epoch - 1, prev), (fork_epoch, cur), (fork_epoch + 5, cur), (0, prev)):
        data = random_data(rng, target_epoch=te)
        want = A.sha(A.attestation_data_root(data) + A.compute_domain(1, version, GVR))
        assert A.signing_root(data, FORK, GVR) == want


def small_cache(n=13_000, epoch=3):   # 3 committees per slot
    ssz = bytearray(beacon_state_deneb_ssz(n, seed=3, n_votes=1, n_hist_roots=1, n_summaries=1))
    CS.set_slot(ssz, epoch * 32 + 5)
    return CS.committee_cache(CS.State(bytes(ssz)), epoch)


def test_one_case_per_status_in_the_reference_order():
    c = small_cache()
    epoch, cps = c["epoch"], c["committees_per_slot"]
    assert cps == 3
    slot = epoch * 32 + 7
    members = A.committee((epoch, c["shuffling"], cps), slot, 1)
    sig = bytes(96)
    full = np.ones(len(members), dtype=np.uint8)
    data = attestation_data_ssz(slot, 1, bytes(32), (epoch - 1, bytes(32)), (epoch, bytes(32)))
    ok_ssz = attestation_ssz(full, data, sig)

    def idx(ssz, electra=False, table_len=1 << 40):
        return A.index_attestation(ssz, electra, [c], table_len, FORK, GVR)

    st, got, root = idx(ok_ssz)
    assert st == A.OK and got.tolist() == sorted(members.tolist()) and root == A.signing_root(data, FORK, GVR)
    # MALFORMED: a wrong offset, no delimiter, too many bits, a short record
    assert idx(b"\x00\x00\x00\x00" + ok_ssz[4:])[0] == A.MALFORMED
    assert idx(ok_ssz[:-1] + b"\x00")[0] == A.MALFORMED
    assert idx(attestation_ssz(np.ones(2049, dtype=np.uint8), data, sig))[0] == A.MALFORMED
    assert idx(ok_ssz[:228])[0] == A.MALFORMED
    # NO_CACHE beats NO_COMMITTEE and BITFIELD_LENGTH
    other = attestation_data_ssz(slot + 32, 99, bytes(32), (epoch, bytes(32)), (epoch + 1, bytes(32)))
    assert idx(attestation_ssz(np.ones(3, dtype=np.uint8), other, sig))[0] == A.NO_CACHE
    # NO_COMMITTEE beats BITFIELD_LENGTH
    bad_index = attestation_data_ssz(slot, cps, bytes(32), (epoch - 1, bytes(32)), (epoch, bytes(32)))
    assert idx(attestation_ssz(np.ones(3, dtype=np.uint8), bad_index, sig))[0] == A.NO_COMMITTEE
    assert idx(attestation_ssz(full[:-1], data, sig))[0] == A.BITFIELD_LENGTH
    # UNKNOWN_VALIDATOR: an attester beyond the table
    assert idx(ok_ssz, table_len=int(members.max()))[0] == A.UNKNOWN_VALIDATOR
    assert idx(ok_ssz, table_len=int(members.max()) + 1)[0] == A.OK
    # Electra: committees in ascending order; an index beyond the slot's committees first, then the summed length
    edata = attestation_data_ssz(slot, 0, bytes(32), (epoch - 1, bytes(32)), (epoch, bytes(32)))
    m0, m2 = (A.committee((epoch, c["shuffling"], cps), slot, k) for k in (0, 2))
    both = np.ones(len(m0) + len(m2), dtype=np.uint8)
    st, got, _ = idx(attestation_ssz(both, edata, sig, 0b101), electra=True)
    assert st == A.OK and got.tolist() == sorted(m0.tolist() + m2.tolist())
    assert idx(attestation_ssz(both, edata, sig, 0b101 | (1 << cps)), electra=True)[0] == A.NO_COMMITTEE
    assert idx(attestation_ssz(both[:-1], edata, sig, 0b101), electra=True)[0] == A.BITFIELD_LENGTH
    st, got, _ = idx(attestation_ssz([], edata, sig, 0), electra=True)   # no committee: an empty set, not an error
    assert st == A.OK and len(got) == 0
    assert idx(ok_ssz, electra=True)[0] == A.MALFORMED   # a pre-Electra encoding is not an Electra one


def test_restatement_agrees_with_the_committee_cache_getters():
    c = small_cache()
    cc = CommitteeCache(c["epoch"], c["shuffling"], c["positions"], c["committees_per_slot"], c["seed"])
    for slot, index, members in CS.committees(c)[::7]:
        assert np.array_equal(A.committee(A.spec_cache(cc), slot, index), members)
        assert np.array_equal(cc.get_beacon_committee(slot, index).committee, members)


@pytest.mark.parametrize("electra", [False, True])
def test_mainnet_genesis_single_bit_attestations_cover_every_validator_once(electra):
    ssz, meta = genesis_state("mainnet")
    c = CS.committee_cache(CS.State(ssz), 0)
    seen = []
    for slot, index, members in CS.committees(c):
        data = attestation_data_ssz(slot, 0 if electra else index, bytes(32), (0, bytes(32)), (0, bytes(32)))
        for pos in range(len(members)):
            bits = np.zeros(len(members), dtype=np.uint8)
            bits[pos] = 1
            att = attestation_ssz(bits, data, bytes(96), (1 << index) if electra else None)
            st, got, _ = A.index_attestation(att, electra, [c], meta["n_validators"], FORK, GVR)
            assert st == A.OK and len(got) == 1
            seen.append(int(got[0]))
    assert sorted(seen) == list(range(meta["n_validators"]))
    assert struct.unpack_from("<Q", ssz, CS.O_SLOT)[0] == 0
