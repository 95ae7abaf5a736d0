"""CPU-only: the host grouping of signature sets by message (lhb200_debug_group_messages, the function the batch
uploads run) against a Python dict: groups in order of first occurrence, members ascending, all 32 bytes compared."""
import numpy as np
import pytest

from lighthouse_b200 import bls


def dict_grouping(msgs):
    groups = {}
    for i in range(len(msgs) // 32):
        groups.setdefault(msgs[32 * i:32 * i + 32], []).append(i)
    members = [i for g in groups.values() for i in g]
    offsets = np.concatenate([[0], np.cumsum([len(g) for g in groups.values()])])
    return np.array(members, dtype=np.uint32), offsets.astype(np.uint32)


def check(msgs):
    members, offsets = bls.group_messages(msgs)
    want_members, want_offsets = dict_grouping(msgs)
    np.testing.assert_array_equal(offsets, want_offsets)
    np.testing.assert_array_equal(members, want_members)
    # first-occurrence order and ascending members, stated directly
    firsts = members[offsets[:-1]]
    assert (np.diff(firsts.astype(np.int64)) > 0).all()
    for g in range(len(offsets) - 1):
        assert (np.diff(members[offsets[g]:offsets[g + 1]].astype(np.int64)) > 0).all()
    return len(offsets) - 1


@pytest.mark.parametrize("n,k", [(2, 1), (2, 2), (64, 1), (64, 4), (64, 16), (64, 64), (1000, 3), (1000, 999),
                                 (5000, 40), (20000, 2048), (20000, 20000)])
def test_random_batches_match_dict(n, k):
    rng = np.random.default_rng(n * 7919 + k)
    pool = rng.integers(0, 256, size=(k, 32), dtype=np.uint8)
    pick = rng.integers(0, k, size=n)
    pick[rng.permutation(n)[:k]] = np.arange(k)      # every pool message occurs
    msgs = pool[pick].tobytes()
    assert check(msgs) == k


@pytest.mark.parametrize("prefix", [8, 16, 31])
def test_shared_prefixes_are_distinct(prefix):
    """messages equal in their first 8, 16 or 31 bytes (and in their fingerprint words' prefix) stay apart"""
    rng = np.random.default_rng(prefix)
    base = rng.integers(0, 256, size=32, dtype=np.uint8)
    k = 200 if prefix < 31 else 256
    pool = np.repeat(base[None], k, axis=0)
    if prefix < 31:
        pool[:, prefix:] = rng.integers(0, 256, size=(k, 32 - prefix), dtype=np.uint8)
    else:
        pool[:, 31] = np.arange(k, dtype=np.uint8)
    assert len({bytes(r) for r in pool}) == k
    pick = np.concatenate([np.arange(k), rng.integers(0, k, size=3 * k)])
    rng.shuffle(pick)
    assert check(pool[pick].tobytes()) == k


def test_all_identical():
    msgs = bytes(range(32)) * 777
    members, offsets = bls.group_messages(msgs)
    assert list(offsets) == [0, 777] and list(members) == list(range(777))


def test_all_distinct():
    rng = np.random.default_rng(3)
    msgs = rng.integers(0, 256, size=(3000, 32), dtype=np.uint8)
    msgs[:, :4] = np.arange(3000, dtype=np.uint32).view(np.uint8).reshape(3000, 4)   # surely distinct
    members, offsets = bls.group_messages(msgs.tobytes())
    assert list(offsets) == list(range(3001)) and list(members) == list(range(3000))


def test_single_set():
    members, offsets = bls.group_messages(bytes(32))
    assert list(offsets) == [0, 1] and list(members) == [0]
