"""From-spec restatement of committees, proposers and the next sync committee over decoded BeaconState bytes (no GPU):
the active set, get_seed, CommitteeCache::initialized with its committee ranges, compute_proposer_index and
get_next_sync_committee_indices (consensus-specs phase0 / altair beacon-chain; the reference's
committee_cache.rs:64-125,313-373 and beacon_state.rs:890-936,1025-1125,1507-1536), mainnet preset.  hashlib and numpy
only, except the shuffle, which is the pinned C oracle's shuffle_list."""
import hashlib
import struct

import numpy as np

from tests import oracle_lib as O

SLOTS_PER_EPOCH, SHUFFLE_ROUND_COUNT, MAX_COMMITTEES_PER_SLOT, TARGET_COMMITTEE_SIZE = 32, 90, 64, 128
EPOCHS_PER_HISTORICAL_VECTOR, MIN_SEED_LOOKAHEAD = 65536, 1
MAX_EFFECTIVE_BALANCE, MAX_RANDOM_BYTE, SYNC_COMMITTEE_SIZE = 32_000_000_000, 255, 512
DOMAIN_BEACON_PROPOSER, DOMAIN_BEACON_ATTESTER, DOMAIN_SYNC_COMMITTEE = 0, 1, 7
# BeaconState fixed-part offsets, the same in every fork: slot, the validators offset, randao_mixes
O_SLOT, O_VAL_OFF, O_RANDAO = 40, 524552, 524560
VALIDATOR_BYTES = 121


class EpochOutOfBounds(ValueError):
    pass


class InsufficientValidators(ValueError):
    pass


def sha(b):
    return hashlib.sha256(b).digest()


class State:
    """What the committee functions read from a BeaconState's SSZ: the slot, the validator records, randao_mixes."""

    def __init__(self, ssz):
        self.slot = struct.unpack_from("<Q", ssz, O_SLOT)[0]
        lo, hi = struct.unpack_from("<II", ssz, O_VAL_OFF)
        self.validators = np.frombuffer(ssz[lo:hi], dtype=np.uint8).reshape(-1, VALIDATOR_BYTES)
        self.randao_mixes = bytes(ssz[O_RANDAO:O_RANDAO + 32 * EPOCHS_PER_HISTORICAL_VECTOR])

    @property
    def current_epoch(self):
        return self.slot // SLOTS_PER_EPOCH

    def field(self, off):
        return np.ascontiguousarray(self.validators[:, off:off + 8]).view("<u8").reshape(-1)

    def effective_balance(self, i):
        return int.from_bytes(bytes(self.validators[i, 80:88]), "little")

    def min_randao_epoch(self):
        return max(self.current_epoch + 1 - EPOCHS_PER_HISTORICAL_VECTOR, 0)


def active_indices(state, epoch):
    """Indices with activation_epoch <= epoch < exit_epoch, ascending."""
    act, exit_ = state.field(97), state.field(105)
    return np.nonzero((act <= np.uint64(epoch)) & (np.uint64(epoch) < exit_))[0].astype(np.uint64)


def get_seed(state, epoch, domain):
    i = (epoch + EPOCHS_PER_HISTORICAL_VECTOR - MIN_SEED_LOOKAHEAD - 1) % EPOCHS_PER_HISTORICAL_VECTOR
    return sha(struct.pack("<IQ", domain, epoch) + state.randao_mixes[32 * i:32 * i + 32])


class ShuffledIndex:
    """compute_shuffled_index(index, n, seed, 90) with its pivots and source hashes memoised for one (n, seed)."""

    def __init__(self, n, seed, rounds=SHUFFLE_ROUND_COUNT):
        self.n, self.seed, self.rounds = n, seed, rounds
        self.pivots = [int.from_bytes(sha(seed + bytes([r]))[:8], "little") % n for r in range(rounds)]
        self.sources = {}

    def __call__(self, index):
        n = self.n
        for r in range(self.rounds):
            flip = (self.pivots[r] + n - index) % n
            pos = max(index, flip)
            key = (r, pos >> 8)
            if key not in self.sources:
                self.sources[key] = sha(self.seed + bytes([r]) + (pos >> 8).to_bytes(4, "little"))
            if (self.sources[key][(pos % 256) // 8] >> (pos % 8)) & 1:
                index = flip
        return index


def compute_shuffled_index(index, n, seed, rounds=SHUFFLE_ROUND_COUNT):
    return ShuffledIndex(n, seed, rounds)(index)


def committees_per_slot(n_active):
    return max(1, min(MAX_COMMITTEES_PER_SLOT, n_active // SLOTS_PER_EPOCH // TARGET_COMMITTEE_SIZE))


def committee_range(epoch_committee_count, index_in_epoch, n):
    if epoch_committee_count == 0 or index_in_epoch >= epoch_committee_count:
        return None
    return n * index_in_epoch // epoch_committee_count, n * (index_in_epoch + 1) // epoch_committee_count


def committee_cache(state, epoch):
    """CommitteeCache::initialized -> dict(epoch, seed, shuffling, positions, committees_per_slot)."""
    if max(epoch - 2, 0) < state.min_randao_epoch() or epoch > state.current_epoch + 1:
        raise EpochOutOfBounds(epoch)
    active = active_indices(state, epoch)
    if len(active) == 0:
        raise InsufficientValidators(epoch)
    seed = get_seed(state, epoch, DOMAIN_BEACON_ATTESTER)
    shuffling = np.array(O.shuffle_list(active, SHUFFLE_ROUND_COUNT, seed, False), dtype=np.uint64)
    positions = np.zeros(len(state.validators), dtype=np.uint32)
    positions[shuffling.astype(np.int64)] = np.arange(1, len(shuffling) + 1, dtype=np.uint32)
    return {"epoch": epoch, "seed": seed, "shuffling": shuffling, "positions": positions,
            "committees_per_slot": committees_per_slot(len(active))}


def committees(cache):
    """Every committee of the cache's epoch as (slot, index, members), in slot then index order."""
    cps, n = cache["committees_per_slot"], len(cache["shuffling"])
    out = []
    for k in range(cps * SLOTS_PER_EPOCH):
        lo, hi = committee_range(cps * SLOTS_PER_EPOCH, k, n)
        out.append((cache["epoch"] * SLOTS_PER_EPOCH + k // cps, k % cps, cache["shuffling"][lo:hi]))
    return out


def sample(state, indices, seed, want):
    """The first `want` candidates that pass the effective-balance test (compute_proposer_index when want == 1)."""
    n = len(indices)
    if n == 0:
        raise InsufficientValidators()
    csi = ShuffledIndex(n, seed)
    out, i, rand = [], 0, b""
    while len(out) < want:
        cand = int(indices[csi(i % n)])
        if i % 32 == 0:
            rand = sha(seed + struct.pack("<Q", i // 32))
        if state.effective_balance(cand) * MAX_RANDOM_BYTE >= MAX_EFFECTIVE_BALANCE * rand[i % 32]:
            out.append(cand)
        i += 1
    return out


def beacon_proposer_indices(state):
    epoch = state.current_epoch
    indices = active_indices(state, epoch)
    base = get_seed(state, epoch, DOMAIN_BEACON_PROPOSER)
    return [sample(state, indices, sha(base + struct.pack("<Q", slot)), 1)[0]
            for slot in range(epoch * SLOTS_PER_EPOCH, (epoch + 1) * SLOTS_PER_EPOCH)]


def next_sync_committee_indices(state):
    epoch = state.current_epoch + 1
    return sample(state, active_indices(state, epoch), get_seed(state, epoch, DOMAIN_SYNC_COMMITTEE), SYNC_COMMITTEE_SIZE)


# ---- test helpers: edit the records and fields of a state's SSZ in place (bytearray) -------------------------------
def set_slot(ssz, slot):
    struct.pack_into("<Q", ssz, O_SLOT, slot)


def validators_offset(ssz):
    return struct.unpack_from("<I", ssz, O_VAL_OFF)[0]


def set_validator_u64(ssz, i, field_off, value):
    struct.pack_into("<Q", ssz, validators_offset(ssz) + VALIDATOR_BYTES * i + field_off, value)


def vary_validators(ssz, epoch, rng, share=0.3):
    """Pending activations, exits at and around `epoch`, and many low effective balances on a share of the records."""
    n = (struct.unpack_from("<I", ssz, O_VAL_OFF + 4)[0] - validators_offset(ssz)) // VALIDATOR_BYTES
    for i in rng.choice(n, size=int(n * share), replace=False).tolist():
        kind = int(rng.integers(0, 5))
        if kind == 0:       # activation pending, or activating right at the epoch
            set_validator_u64(ssz, i, 97, epoch + int(rng.integers(-1, 3)) if epoch else int(rng.integers(0, 3)))
        elif kind == 1:     # exiting at, just before or just after the epoch
            set_validator_u64(ssz, i, 105, max(epoch + int(rng.integers(-1, 3)), 0))
        else:               # low effective balance: rejected by most random bytes
            set_validator_u64(ssz, i, 80, int(rng.integers(0, 32)) * 1_000_000_000 // 4)
