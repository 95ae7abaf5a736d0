"""CPU-only: the committee restatement of tests/committee_spec.py pinned by the properties the reference's own tests
check (consensus/types/src/beacon_state/committee_cache/tests.rs), by an independent compute_shuffled_index, and on the
mainnet genesis state; and the lighthouse_b200.committees.CommitteeCache getters over the restatement's arrays."""
import hashlib

import numpy as np
import pytest

from lighthouse_b200.committees import CommitteeCache, CommitteeCacheError
from lighthouse_b200.synthetic import beacon_state_deneb_ssz
from tests import committee_spec as CS
from tests import oracle_lib as O
from tests.phase0_state import genesis_state
from tests.test_shuffle import py_csi


def state_at(n, epoch, seed=5, fork="altair"):
    ssz = bytearray(beacon_state_deneb_ssz(n, seed=seed, fork=fork, n_votes=0, n_hist_roots=0))
    CS.set_slot(ssz, epoch * 32 + 7)
    return ssz


def product_cache(c):
    return CommitteeCache(c["epoch"], c["shuffling"], c["positions"], c["committees_per_slot"], c["seed"])


def test_compute_shuffled_index_matches_the_pinned_ones():
    for n in (1, 2, 33, 300, 1000):
        seed = hashlib.sha256(b"csi-%d" % n).digest()
        csi = CS.ShuffledIndex(n, seed)
        for i in range(0, n, max(1, n // 40)):
            assert csi(i) == py_csi(i, n, seed, 90) == O.compute_shuffled_index(i, n, seed, 90)


def test_default_cache_has_nothing():
    c = CommitteeCache()
    assert not c.is_initialized_at(0)
    assert len(c.active_validator_indices()) == 0
    assert c.get_beacon_committee(0, 0) is None
    assert c.get_attestation_duties(0) is None
    assert c.active_validator_count() == 0 and c.epoch_committee_count() == 0
    with pytest.raises(CommitteeCacheError):
        c.get_beacon_committees_at_slot(0)
    with pytest.raises(CommitteeCacheError):
        c.get_all_beacon_committees()


def test_caches_initialise_at_their_epochs_with_distinct_seeds_and_accurate_positions():
    epoch = 6
    st = CS.State(bytes(state_at(300, epoch)))
    assert st.current_epoch == epoch
    seeds = []
    for e in (epoch - 1, epoch, epoch + 1):
        c = CS.committee_cache(st, e)
        pc = product_cache(c)
        assert pc.is_initialized_at(e) and not pc.is_initialized_at(e + 1)
        active = CS.active_indices(st, e)
        assert list(c["shuffling"]) == O.shuffle_list(active, 90, c["seed"], False)
        assert list(c["shuffling"]) == [int(active[py_csi(i, len(active), c["seed"], 90)]) for i in range(len(active))]
        for i, v in enumerate(c["shuffling"].tolist()):
            assert pc.shuffled_position(v) == i
        seeds.append(c["seed"])
    assert len(set(seeds)) == 3
    for e in range(0, epoch + 2):   # historic epochs build too (lighthouse issue 3270)
        assert CS.committee_cache(st, e)["epoch"] == e
    with pytest.raises(CS.EpochOutOfBounds):
        CS.committee_cache(st, epoch + 2)


def test_min_randao_epoch_boundary():
    current = 2 * 65536
    st = CS.State(bytes(state_at(64, current)))
    m = st.min_randao_epoch()
    assert m == current + 1 - 65536
    CS.committee_cache(st, m + 2)
    with pytest.raises(CS.EpochOutOfBounds):
        CS.committee_cache(st, m + 1)


def test_no_active_validator_is_refused():
    ssz = state_at(40, 3)
    for i in range(40):
        CS.set_validator_u64(ssz, i, 97, 100)
    st = CS.State(bytes(ssz))
    with pytest.raises(CS.InsufficientValidators):
        CS.committee_cache(st, 3)
    with pytest.raises(CS.InsufficientValidators):
        CS.beacon_proposer_indices(st)


def test_product_getters_follow_the_restatement():
    rng = np.random.default_rng(3)
    ssz = state_at(9000, 40)
    CS.vary_validators(ssz, 40, rng)
    st = CS.State(bytes(ssz))
    c = CS.committee_cache(st, 40)
    pc = product_cache(c)
    assert pc.committees_per_slot() == c["committees_per_slot"] == 2
    want = CS.committees(c)
    got = pc.get_all_beacon_committees()
    assert len(got) == len(want) == pc.epoch_committee_count()
    for g, (slot, index, members) in zip(got, want):
        assert (g.slot, g.index) == (slot, index) and list(g.committee) == list(members)
    assert pc.get_beacon_committee(40 * 32 + 3, 2) is None            # index >= committees_per_slot
    assert pc.get_beacon_committee(41 * 32, 0) is None                 # another epoch
    for slot, index, members in want[::7]:
        for pos, v in enumerate(members.tolist()):
            d = pc.get_attestation_duties(v)
            assert (d.slot, d.index, d.committee_position, d.committee_len, d.committees_at_slot) == \
                (slot, index, pos, len(members), 2)
    inactive = [v for v in range(len(st.validators)) if c["positions"][v] == 0]
    assert inactive and all(pc.get_attestation_duties(v) is None for v in inactive[:50])
    assert pc.shuffled_position(len(st.validators)) is None


def test_samplers_on_low_balances():
    """Many low effective balances: the proposer and sync draws reject candidates, and every winner is active."""
    rng = np.random.default_rng(8)
    ssz = state_at(2000, 12)
    CS.vary_validators(ssz, 12, rng, share=0.8)
    st = CS.State(bytes(ssz))
    props = CS.beacon_proposer_indices(st)
    assert len(props) == 32 and set(props) <= set(CS.active_indices(st, 12).tolist())
    sync = CS.next_sync_committee_indices(st)
    assert len(sync) == 512 and set(sync) <= set(CS.active_indices(st, 13).tolist())


def test_mainnet_genesis_committees():
    ssz, meta = genesis_state("mainnet")
    st = CS.State(ssz)
    assert st.slot == 0 and len(st.validators) == meta["n_validators"] == 21063
    assert len(CS.active_indices(st, 0)) == 21063
    for epoch in (0, 1):
        c = CS.committee_cache(st, epoch)
        assert c["committees_per_slot"] == 5
        members = np.concatenate([m for _, _, m in CS.committees(c)])
        assert sorted(members.tolist()) == list(range(21063))   # every validator in exactly one committee
        pc = product_cache(c)
        for slot, index, m in CS.committees(c)[::11]:
            for pos, v in enumerate(m.tolist()[::13]):
                d = pc.get_attestation_duties(v)
                assert (d.slot, d.index, d.committee_position, d.committee_len) == (slot, index, 13 * pos, len(m))
