"""Committees, proposers and the next sync committee from a resident BeaconState (lhb200_state_committee_cache,
lhb200_state_beacon_proposer_indices, lhb200_state_next_sync_committee_indices) against the from-spec restatement of
tests/committee_spec.py, whose shuffle is the pinned C oracle: every fork, the genesis states, sizes that cover 1 to 64
committees per slot, the randao window, the warm path with patches, appends and clones, and the refusals.  The test
without a device runs in the CPU suite."""
import ctypes as C
import struct

import numpy as np
import pytest

from lighthouse_b200.synthetic import beacon_state_deneb_ssz, validators_ssz
from tests import committee_spec as CS
from tests.phase0_state import genesis_state
from tests.test_state_lists_gpu import StateModel, apply, patch, resident

FAR_FUTURE = (1 << 64) - 1


def state_ssz(n, epoch, fork="deneb", seed=11, vary=True):
    ssz = bytearray(beacon_state_deneb_ssz(n, seed=seed, fork=fork, n_votes=3, n_hist_roots=5, n_summaries=2))
    CS.set_slot(ssz, epoch * 32 + 9)
    if vary:
        CS.vary_validators(ssz, epoch, np.random.default_rng(seed + n))
    return bytes(ssz)


def check(h, ssz, epochs=None, samplers=True):
    """The handle's caches at `epochs` (default: previous, current, next), proposers and sync draw == the restatement."""
    s = CS.State(ssz)
    cur = s.current_epoch
    for e in epochs if epochs is not None else sorted({max(cur - 1, 0), cur, cur + 1}):
        want = CS.committee_cache(s, e)
        got = h.committee_cache(e)
        assert got.is_initialized_at(e)
        assert np.array_equal(got.shuffling(), want["shuffling"]), e
        assert np.array_equal(got._positions, want["positions"]), e
        assert got.committees_per_slot() == want["committees_per_slot"]
        assert got.seed == want["seed"]
    if samplers:
        assert h.beacon_proposer_indices() == CS.beacon_proposer_indices(s)
        assert h.next_sync_committee_indices() == CS.next_sync_committee_indices(s)


def launches():
    from lighthouse_b200 import _ffi
    return _ffi.lib.lhb200_launch_count()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["base", "altair", "deneb", "electra"])
def test_forks(gpu, fork):
    from lighthouse_b200 import tree_hash as T
    ssz = state_ssz(3000, 100, fork)
    h = T.ResidentState(ssz, fork)
    check(h, ssz)
    h.release()


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["mainnet", "sepolia"])
def test_genesis_states(gpu, net):
    from lighthouse_b200 import tree_hash as T
    ssz, meta = genesis_state(net)
    h = T.ResidentState(ssz, "base")
    check(h, ssz, epochs=[0, 1])
    c = h.committee_cache(0)
    assert c.active_validator_count() == meta["n_validators"]
    if net == "mainnet":
        assert c.committees_per_slot() == 5
    h.release()


@pytest.mark.gpu
@pytest.mark.parametrize("n,cps", [(1, 1), (31, 1), (4095, 1), (4096, 1), (131_072, 32), (262_144, 64), (500_000, 64)])
def test_sizes(gpu, n, cps):
    from lighthouse_b200 import tree_hash as T
    ssz = state_ssz(n, 300, vary=False)
    h = T.ResidentState(ssz, "deneb")
    assert h.committee_cache(300).committees_per_slot() == cps
    check(h, ssz, epochs=[300, 301] if n >= 100_000 else None)
    h.release()


@pytest.mark.gpu
def test_randao_window_and_refusals_leave_the_handle(gpu):
    from lighthouse_b200 import _ffi, tree_hash as T
    current = 2 * 65536 + 5
    ssz = state_ssz(700, current)
    h = T.ResidentState(ssz, "deneb")
    before = h.root(want_field_roots=True)
    m = current + 1 - 65536
    check(h, ssz, epochs=[m + 2, current - 1, current, current + 1], samplers=False)
    for e in (m + 1, m, 0, current + 2, current + 100):
        with pytest.raises(_ffi.Lhb200Error) as exc:
            h.committee_cache(e)
        assert exc.value.code == _ffi.EINVAL and b"out of bounds" in _ffi.lib.lhb200_last_error()
    assert h.root(want_field_roots=True) == before
    h.release()


@pytest.mark.gpu
def test_warm_path_follows_the_bytes(gpu):
    """Patches to randao_mixes, the slot and validator epochs; an append of inactive validators on the converted handle
    (the positions cover them); a clone, checked again after its source is released."""
    rng = np.random.default_rng(5)
    epoch = 400
    model = StateModel(state_ssz(6000, epoch), "deneb")
    h = resident(model)
    check(h, model.ssz())
    mix = (epoch + 65534) % 65536
    patch(h, model, CS.O_RANDAO + 32 * mix, 0, rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
    check(h, model.ssz())
    patch(h, model, CS.O_SLOT, 0, struct.pack("<Q", (epoch + 1) * 32 + 3))      # the next epoch
    check(h, model.ssz())
    for i in rng.choice(6000, size=40, replace=False).tolist():
        patch(h, model, "validators", 121 * i + 97, struct.pack("<Q", epoch + 2))   # pending at the new epoch
        patch(h, model, "validators", 121 * ((i + 1) % 6000) + 105, struct.pack("<Q", epoch + 1))   # exits at it
    patch(h, model, "validators", 121 * 7 + 80, struct.pack("<Q", 0))
    check(h, model.ssz())
    k = 17
    vals = bytearray(validators_ssz(k, rng))
    for j in range(k):
        vals[121 * j + 97:121 * j + 105] = struct.pack("<Q", FAR_FUTURE)
    n = model.length("validators")
    apply(h, model, [("validators", n + k, n, bytes(vals)),
                     ("balances", n + k, n, np.full(k, 32_000_000_000, dtype="<u8").tobytes()),
                     ("previous_epoch_participation", n + k, n, bytes(k)),
                     ("current_epoch_participation", n + k, n, bytes(k)),
                     ("inactivity_scores", n + k, n, bytes(8 * k))])
    assert h.list_len("validators") == n + k
    c = h.committee_cache(epoch + 1)
    assert len(c._positions) == n + k and not c._positions[n:].any()
    check(h, model.ssz())
    clone = h.clone()
    check(clone, model.ssz())
    h.release()
    check(clone, model.ssz())
    clone.release()


@pytest.mark.gpu
def test_shuffling_matches_shuffle_list(gpu):
    from lighthouse_b200 import tree_hash as T
    from lighthouse_b200.shuffle import shuffle_list
    ssz = state_ssz(20_000, 77, "electra")
    s = CS.State(ssz)
    h = T.ResidentState(ssz, "electra")
    for e in (76, 77, 78):
        active = CS.active_indices(s, e)
        c = h.committee_cache(e)
        assert c.seed == CS.get_seed(s, e, CS.DOMAIN_BEACON_ATTESTER)
        assert c.shuffling().tolist() == shuffle_list(active, 90, c.seed, False)
    h.release()


@pytest.mark.gpu
def test_calls_only_read_a_handle_with_pending_edits(gpu):
    from lighthouse_b200 import tree_hash as T
    model = StateModel(state_ssz(5000, 60, "capella"), "capella")
    h = resident(model)
    patch(h, model, "validators", 121 * 3 + 97, struct.pack("<Q", 61))
    patch(h, model, CS.O_SLOT, 0, struct.pack("<Q", 60 * 32 + 31))
    h.committee_cache(60)
    h.beacon_proposer_indices()
    h.next_sync_committee_indices()
    fresh = T.ResidentState(model.ssz(), "capella")
    assert h.root(want_field_roots=True) == fresh.root(want_field_roots=True)
    check(h, model.ssz())
    assert h.root(want_field_roots=True) == fresh.root(want_field_roots=True)
    fresh.release()
    h.release()


@pytest.mark.gpu
def test_launch_count_does_not_depend_on_the_validator_count(gpu):
    from lighthouse_b200 import tree_hash as T
    counts = []
    for n in (4096, 500_000):
        h = T.ResidentState(state_ssz(n, 50, vary=False), "deneb")
        per = []
        for call in (lambda: h.committee_cache(50), h.beacon_proposer_indices, h.next_sync_committee_indices):
            call()
            l0 = launches()
            call()
            per.append(launches() - l0)
        counts.append(per)
        h.release()
    assert counts[0] == counts[1] == [6, 4, 4]


@pytest.mark.gpu
def test_refusals(gpu):
    from lighthouse_b200 import _ffi, tree_hash as T
    ssz = state_ssz(300, 9)
    h = T.ResidentState(ssz, "deneb")
    out = np.zeros(512, dtype=np.uint64)
    pos = np.zeros(300, dtype=np.uint32)
    info = _ffi.CommitteeInfo()
    assert _ffi.lib.lhb200_state_committee_cache(h._h, 9, out.ctypes.data, pos.ctypes.data, 299, C.byref(info)) == _ffi.EINVAL
    assert b"cap" in _ffi.lib.lhb200_last_error()
    assert _ffi.lib.lhb200_state_committee_cache(h._h, 9, out.ctypes.data, None, 300, C.byref(info)) == _ffi.OK
    h.release()
    sh = T.ShardedState(beacon_state_deneb_ssz(4096, seed=2), 0, 2)
    assert _ffi.lib.lhb200_state_committee_cache(sh._h, 0, out.ctypes.data, None, 1 << 20, C.byref(info)) == _ffi.EINVAL
    assert _ffi.lib.lhb200_state_beacon_proposer_indices(sh._h, out.ctypes.data) == _ffi.EINVAL
    assert _ffi.lib.lhb200_state_next_sync_committee_indices(sh._h, out.ctypes.data) == _ffi.EINVAL
    assert b"sharded" in _ffi.lib.lhb200_last_error()
    sh.release()
    none = bytearray(ssz)
    for i in range(300):
        CS.set_validator_u64(none, i, 97, FAR_FUTURE)
    h = T.ResidentState(bytes(none), "deneb")
    before = h.root(want_field_roots=True)
    for call in (lambda: h.committee_cache(9), h.beacon_proposer_indices, h.next_sync_committee_indices):
        with pytest.raises(_ffi.Lhb200Error) as exc:
            call()
        assert exc.value.code == _ffi.EINVAL and b"no validator is active" in _ffi.lib.lhb200_last_error()
    assert h.root(want_field_roots=True) == before
    h.release()


def test_no_device_gives_enodev():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    out = np.zeros(512, dtype=np.uint64)
    info = _ffi.CommitteeInfo()
    assert _ffi.lib.lhb200_state_committee_cache(None, 0, out.ctypes.data, None, 512, C.byref(info)) == _ffi.ENODEV
    assert _ffi.lib.lhb200_state_beacon_proposer_indices(None, out.ctypes.data) == _ffi.ENODEV
    assert _ffi.lib.lhb200_state_next_sync_committee_indices(None, out.ctypes.data) == _ffi.ENODEV
