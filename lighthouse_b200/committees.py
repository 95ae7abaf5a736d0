"""CommitteeCache (consensus/types/src/beacon_state/committee_cache.rs) over the arrays the device computes from a
resident BeaconState (lhb200_state_committee_cache; ResidentState.committee_cache).  The getters are plain index
arithmetic over the shuffling, as in the reference (committee_cache.rs:140-355); no hashing happens here.
"""
from collections import namedtuple

import numpy as np

SLOTS_PER_EPOCH = 32

BeaconCommittee = namedtuple("BeaconCommittee", "slot index committee")
AttestationDuty = namedtuple("AttestationDuty", "slot index committee_position committee_len committees_at_slot")


class CommitteeCacheError(ValueError):
    """The reference's committee_cache errors: CommitteeCacheUninitialized and NoCommittee."""


def compute_committee_range_in_epoch(epoch_committee_count, index_in_epoch, shuffling_len):
    """committee_cache.rs:313-330: (start, end) of the index_in_epoch'th committee, None when out of range."""
    if epoch_committee_count == 0 or index_in_epoch >= epoch_committee_count:
        return None
    return (shuffling_len * index_in_epoch // epoch_committee_count,
            shuffling_len * (index_in_epoch + 1) // epoch_committee_count)


class CommitteeCache:
    """CommitteeCache::initialized(state, epoch) as computed on the device, or the default (uninitialised) cache.
    shuffling: the active indices in shuffled order; positions: per validator 0 (None) or position + 1."""

    def __init__(self, epoch=None, shuffling=(), positions=(), committees_per_slot=0, seed=None):
        self.initialized_epoch = epoch
        self._shuffling = np.asarray(shuffling, dtype=np.uint64)
        self._positions = np.asarray(positions, dtype=np.uint32)
        self._committees_per_slot = int(committees_per_slot)
        self.seed = seed
        self.slots_per_epoch = SLOTS_PER_EPOCH

    def is_initialized_at(self, epoch):
        return self.initialized_epoch is not None and self.initialized_epoch == epoch

    def active_validator_indices(self):
        """The shuffled active indices (not in ascending order); empty when uninitialised."""
        return self._shuffling

    def shuffling(self):
        return self._shuffling

    def active_validator_count(self):
        return len(self._shuffling)

    def committees_per_slot(self):
        return self._committees_per_slot

    def epoch_committee_count(self):
        return self._committees_per_slot * self.slots_per_epoch

    def _committee_range(self, index_in_epoch):
        return compute_committee_range_in_epoch(self.epoch_committee_count(), index_in_epoch, len(self._shuffling))

    def get_beacon_committee(self, slot, index):
        """BeaconCommittee(slot, index, committee), or None when uninitialised, at another epoch or index out of range."""
        if (self.initialized_epoch is None or not self.is_initialized_at(slot // self.slots_per_epoch)
                or index >= self._committees_per_slot):
            return None
        r = self._committee_range((slot % self.slots_per_epoch) * self._committees_per_slot + index)
        if r is None:
            return None
        return BeaconCommittee(slot, index, self._shuffling[r[0]:r[1]])

    def get_beacon_committees_at_slot(self, slot):
        if self.initialized_epoch is None:
            raise CommitteeCacheError("CommitteeCacheUninitialized")
        out = []
        for index in range(self._committees_per_slot):
            c = self.get_beacon_committee(slot, index)
            if c is None:
                raise CommitteeCacheError(f"NoCommittee {{ slot: {slot}, index: {index} }}")
            out.append(c)
        return out

    def get_all_beacon_committees(self):
        if self.initialized_epoch is None:
            raise CommitteeCacheError("CommitteeCacheUninitialized")
        start = self.initialized_epoch * self.slots_per_epoch
        return [c for slot in range(start, start + self.slots_per_epoch) for c in self.get_beacon_committees_at_slot(slot)]

    def shuffled_position(self, validator_index):
        if validator_index < 0 or validator_index >= len(self._positions):
            return None
        p = int(self._positions[validator_index])
        return p - 1 if p else None

    def get_attestation_duties(self, validator_index):
        """AttestationDuty of the validator, or None when it has none (committee_cache.rs:245-280).  Committees split
        the shuffling evenly, so the committee holding position i is found by division and checked against its range."""
        i = self.shuffled_position(validator_index)
        if i is None:
            return None
        count = self.epoch_committee_count()
        n = len(self._shuffling)
        nth = min((i * count) // n, count - 1) if n else 0
        while nth > 0 and self._committee_range(nth)[0] > i:
            nth -= 1
        while self._committee_range(nth)[1] <= i:
            nth += 1
        start, end = self._committee_range(nth)
        slot = self.initialized_epoch * self.slots_per_epoch + nth // self._committees_per_slot
        return AttestationDuty(slot, nth % self._committees_per_slot, i - start, end - start, self._committees_per_slot)


class DeviceCommitteeCache:
    """A committee cache that stays on the device (lhb200_state_committee_cache_create), what
    lighthouse_b200.attestations.verify_attestations reads.  It owns its shuffling and does not depend on the state it
    came from: releasing, patching or cloning that state leaves it as it is."""

    def __init__(self, handle):
        self._h = handle

    @property
    def info(self):
        """lhb200_committee_info: epoch, n_validators, n_active, committees_per_slot, seed."""
        from . import _ffi
        info = _ffi.CommitteeInfo()
        _ffi.check(_ffi.lib.lhb200_committee_cache_info(self._h, _ffi.C.byref(info)), "lhb200_committee_cache_info")
        return info

    @property
    def epoch(self):
        return self.info.epoch

    def to_host(self):
        """The same cache as a CommitteeCache, from one device-to-host copy of the shuffling (the positions are its
        inverse, scattered here)."""
        from . import _ffi
        info = self.info
        shuffling = np.zeros(max(info.n_active, 1), dtype=np.uint64)
        _ffi.check(_ffi.lib.lhb200_committee_cache_shuffling(self._h, shuffling.ctypes.data, len(shuffling)),
                   "lhb200_committee_cache_shuffling")
        shuffling = shuffling[:info.n_active]
        positions = np.zeros(info.n_validators, dtype=np.uint32)
        positions[shuffling.astype(np.int64)] = np.arange(1, info.n_active + 1, dtype=np.uint32)
        return CommitteeCache(info.epoch, shuffling, positions, info.committees_per_slot, bytes(info.seed))

    def release(self):
        if self._h:
            from . import _ffi
            _ffi.lib.lhb200_committee_cache_release(self._h)
            self._h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass
