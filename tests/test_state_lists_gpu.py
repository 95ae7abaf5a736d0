"""Resizable lists of a resident BeaconState (lhb200_state_list_edit, lhb200_state_set_payload_header): a warm handle
follows a chain whose blocks append eth1 votes and deposits, replace the payload header (extra_data changes length)
and whose epochs rotate participation, reset votes, push historical summaries and drain Electra's pending lists.

The expected state is kept as its fixed part plus one byte string per variable-size field, re-joined with recomputed
offsets; Deneb is checked against the C oracle, every fork against the from-spec merkleization of tests/ssz_spec.py."""
import ctypes as C
import struct

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200.synthetic import beacon_state_deneb_ssz, validators_ssz
from tests import oracle_lib as O
from tests import ssz_spec

HEADER_FIXED = {"bellatrix": 536, "capella": 568, "deneb": 584, "electra": 648}


class StateModel:
    """SSZ of a BeaconState as fixed part + the bytes of each variable-size field."""

    def __init__(self, ssz, fork):
        self.fork = fork
        self.typ = S.BEACON_STATE_BY_FORK[fork]
        self.names = [name for name, _ in self.typ[1]]
        self.var, pos = [], 0
        for name, ft in self.typ[1]:
            if S.is_fixed(ft):
                pos += S.fixed_size(ft)
            else:
                self.var.append((name, pos))
                pos += 4
        self.fixed = bytearray(ssz[:pos])
        offs = [struct.unpack_from("<I", ssz, p)[0] for _, p in self.var] + [len(ssz)]
        self.parts = {name: bytearray(ssz[offs[i]:offs[i + 1]]) for i, (name, _) in enumerate(self.var)}

    def ssz(self):
        out, at = bytearray(self.fixed), len(self.fixed)
        for name, pos in self.var:
            out[pos:pos + 4] = struct.pack("<I", at)
            at += len(self.parts[name])
        return bytes(out) + b"".join(bytes(self.parts[n]) for n, _ in self.var)

    def offset(self, name):
        at = len(self.fixed)
        for n, _ in self.var:
            if n == name:
                return at
            at += len(self.parts[n])
        raise KeyError(name)

    def item_bytes(self, name):
        return S.fixed_size(self.typ[1][self.names.index(name)][1][1])

    def length(self, name):
        return len(self.parts[name]) // self.item_bytes(name)

    def edit(self, name, new_len, first, data):
        ib = self.item_bytes(name)
        p = self.parts[name]
        p[first * ib:first * ib + len(data)] = data
        del p[new_len * ib:]
        assert len(p) == new_len * ib


def expected(model):
    ssz = model.ssz()
    if model.fork == "deneb":
        return O.beacon_state_root_deneb(ssz)
    value = ssz_spec.deserialize(model.typ, ssz)
    return ssz_spec.hash_tree_root(model.typ, value), [ssz_spec.hash_tree_root(ft, value[n]) for n, ft in model.typ[1]]


def check(st, model, warm=None, fresh=True):
    from lighthouse_b200 import tree_hash as T
    want, want_fields = expected(model)
    got, fields = st.root(want_field_roots=True)
    bad = [i for i, (g, w) in enumerate(zip(fields, want_fields)) if g != w]
    assert not bad, f"field roots differ: {[model.names[i] for i in bad]}"
    assert got == want
    for name in ("eth1_data_votes", "validators", "balances", "inactivity_scores"):
        assert st.list_len(name) == model.length(name)
    if fresh:
        f = T.ResidentState(model.ssz(), model.fork)
        assert f.root() == got
        assert f.hash_units == st.hash_units
        f.release()
    if warm is True:
        # warm: dirty paths, the changed lists' ladders and mix-ins, and the tail; the tail alone is what a root with
        # nothing dirty computes
        hashes = st.last_root_hashes
        assert st.root() == got
        tail = st.last_root_hashes
        assert hashes - tail < st.hash_units // 20, (hashes, tail, st.hash_units)
        if model.length("validators") >= 20_000:
            assert hashes < st.hash_units // 20, (hashes, st.hash_units)
    elif warm == "bulk":   # thousands of items appended or rewritten on a small state: warm, but no longer a small share
        assert st.last_root_hashes < st.hash_units // 2, (st.last_root_hashes, st.hash_units)
    elif warm is False:
        assert st.last_root_hashes == st.hash_units


def header_bytes(rng, fork, extra_len):
    fixed = HEADER_FIXED[fork]
    h = bytearray(rng.integers(0, 256, size=fixed, dtype=np.uint8).tobytes())
    h[436:440] = struct.pack("<I", fixed)
    return bytes(h) + rng.integers(0, 256, size=extra_len, dtype=np.uint8).tobytes()


def rb(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def raw_edit(st, edits, data=b""):
    """lhb200_state_list_edit with edits given as (field index, new_len, first, n): no checks on the Python side."""
    from lighthouse_b200 import _ffi
    arr = (_ffi.ListEdit * len(edits))(*[_ffi.ListEdit(f, 0, nl, first, n) for f, nl, first, n in edits])
    p = C.create_string_buffer(data, max(len(data), 1))
    return _ffi.lib.lhb200_state_list_edit(st._h, C.cast(arr, C.c_void_p), len(edits), p)


def resident(model):
    from lighthouse_b200 import tree_hash as T
    st = T.ResidentState(model.ssz(), model.fork)
    st.enable_incremental()
    st.root()
    return st


def deposits(rng, model, k):
    """The five per-validator lists (plus pending_balance_deposits from Electra) grow by k together."""
    n = model.length("validators")
    vals = validators_ssz(k, rng)
    edits = [("validators", n + k, n, vals),
             ("balances", n + k, n, np.full(k, 32_000_000_000, dtype="<u8").tobytes()),
             ("previous_epoch_participation", n + k, n, bytes(k)),
             ("current_epoch_participation", n + k, n, bytes(k)),
             ("inactivity_scores", n + k, n, bytes(8 * k))]
    if model.fork == "electra":
        m = model.length("pending_balance_deposits")
        edits.append(("pending_balance_deposits", m + k, m,
                      b"".join(struct.pack("<QQ", n + i, 32_000_000_000) for i in range(k))))
    return edits


def apply(st, model, edits):
    st.list_edit(edits)
    for name, new_len, first, data in edits:
        model.edit(name, new_len, first, data)


def patch(st, model, name_or_off, rel, data):
    """Same-length patch at an offset into the CURRENT encoding (a variable-size field plus `rel`, or a fixed offset)."""
    off = model.offset(name_or_off) + rel if isinstance(name_or_off, str) else name_or_off
    if isinstance(name_or_off, str):
        model.parts[name_or_off][rel:rel + len(data)] = data
    else:
        model.fixed[off:off + len(data)] = data
    st.patch(off, data)


@pytest.mark.gpu
@pytest.mark.parametrize("n_validators", [20_000, 32_760])
def test_chain_replay_deneb(gpu, n_validators):
    """Eight slots: patches into the current encoding interleaved with list edits and header replacements.  32 760 + 16
    deposits crosses a power of two in all five per-validator trees at once."""
    rng = np.random.default_rng(n_validators)
    model = StateModel(beacon_state_deneb_ssz(n_validators, seed=3, n_votes=5, n_summaries=3), "deneb")
    st = resident(model)
    for slot in range(8):
        patch(st, model, 40, 0, struct.pack("<Q", 5000 + slot))                          # slot
        patch(st, model, 524560 + 32 * int(rng.integers(0, 65536)), 0, rb(rng, 32))      # randao mix
        patch(st, model, 176 + 32 * (slot % 8192), 0, rb(rng, 32))                         # block root
        apply(st, model, [("eth1_data_votes", model.length("eth1_data_votes") + 1,
                           model.length("eth1_data_votes"), rb(rng, 72))])
        nv = model.length("validators")
        for vi in rng.choice(nv, size=20, replace=False):                                # validators and balances
            patch(st, model, "validators", 121 * int(vi) + 80, struct.pack("<Q", int(rng.integers(1, 1 << 40))))
            patch(st, model, "balances", 8 * int(vi), struct.pack("<Q", int(rng.integers(1, 1 << 40))))
        c0 = int(rng.integers(0, nv - 300))
        patch(st, model, "current_epoch_participation", c0, bytes(rng.integers(0, 8, size=300, dtype=np.uint8)))
        if slot % 2 == 0:
            apply(st, model, deposits(rng, model, 16))
            patch(st, model, "validators", 121 * (model.length("validators") - 1) + 88, bytes([1]))
        hdr = header_bytes(rng, "deneb", int(rng.integers(0, 33)))
        st.set_payload_header(hdr)
        model.parts["latest_execution_payload_header"][:] = hdr
        patch(st, model, "latest_execution_payload_header", 0, rb(rng, 32))              # parent_hash after a move
        if slot == 5:                                                                      # epoch boundary
            nv = model.length("validators")
            apply(st, model, [("previous_epoch_participation", nv, 0, bytes(model.parts["current_epoch_participation"])),
                              ("current_epoch_participation", nv, 0, bytes(nv)),
                              ("eth1_data_votes", 0, 0, b""),
                              ("historical_summaries", model.length("historical_summaries") + 1,
                               model.length("historical_summaries"), rb(rng, 64))])
            patch(st, model, "balances", 0, rng.integers(1, 1 << 40, size=nv, dtype="<u8").tobytes()[:8 * 4000])
        check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["capella", "electra"])
def test_lists_grow_drain_and_reset(gpu, fork):
    """Pending lists grow, drain from the front, shrink across a power of two and go to 0; historical_summaries
    pushes; eth1 votes go 0 -> 1 -> 2 -> 3 -> 2048, the 2049th is refused, then reset."""
    from lighthouse_b200 import Lhb200Error, _ffi
    rng = np.random.default_rng(11)
    model = StateModel(beacon_state_deneb_ssz(37, seed=9, fork=fork, n_votes=0, n_summaries=0, n_pending=(5, 0, 3)),
                       fork)
    st = resident(model)
    for n in (1, 2, 3, 2048):
        k = model.length("eth1_data_votes")
        apply(st, model, [("eth1_data_votes", n, k, rb(rng, 72 * (n - k)))])
        check(st, model, warm=True if n < 2048 else "bulk")
    with pytest.raises(Lhb200Error) as e:
        st.list_edit([("eth1_data_votes", 2049, 2048, rb(rng, 72))])
    assert e.value.code == _ffi.EINVAL
    for _ in range(2):
        k = model.length("historical_summaries")
        apply(st, model, [("historical_summaries", k + 1, k, rb(rng, 64)), ("eth1_data_votes", 0, 0, b"")])
        check(st, model, warm=True)
    model.parts["latest_execution_payload_header"][:] = header_bytes(rng, fork, 0)   # extra_data emptied
    st.set_payload_header(bytes(model.parts["latest_execution_payload_header"]))
    check(st, model, warm=True)
    if fork == "electra":
        sizes = {"pending_balance_deposits": 16, "pending_partial_withdrawals": 24, "pending_consolidations": 16}
        for name, item in sizes.items():                                   # grow past 1024 items
            k = model.length(name)
            apply(st, model, [(name, 1100, k, rb(rng, item * (1100 - k)))])
        check(st, model, warm="bulk")
        for name, item in sizes.items():                                   # front drain: 1100 -> 1000 -> 700
            for keep in (1000, 700):
                rest = bytes(model.parts[name][item * (model.length(name) - keep):])
                apply(st, model, [(name, keep, 0, rest)])
            check(st, model, warm="bulk")
        apply(st, model, [(n, 3, 3, b"") for n in sizes])                  # truncate across many powers of two
        check(st, model, warm=True)
        apply(st, model, [(n, 0, 0, b"") for n in sizes])                  # empty
        check(st, model, warm=True)
        apply(st, model, [(n, 1, 0, rb(rng, sizes[n])) for n in sizes])    # and one again
        check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
def test_altair_one_round(gpu):
    """Altair: votes and deposits follow; there is no header and no historical_summaries."""
    from lighthouse_b200 import Lhb200Error, _ffi
    rng = np.random.default_rng(5)
    model = StateModel(beacon_state_deneb_ssz(300, seed=2, fork="altair"), "altair")
    st = resident(model)
    apply(st, model, deposits(rng, model, 16) + [("eth1_data_votes", model.length("eth1_data_votes") + 1,
                                                  model.length("eth1_data_votes"), rb(rng, 72))])
    patch(st, model, "balances", 8 * 7, struct.pack("<Q", 99))
    check(st, model, warm=True)
    with pytest.raises(Lhb200Error) as e:
        st.set_payload_header(b"\0" * 536)
    assert e.value.code == _ffi.EINVAL
    assert raw_edit(st, [(27, 1, 0, 1)], rb(rng, 64)) == _ffi.EINVAL           # historical_summaries: not in Altair
    st.release()


@pytest.mark.gpu
def test_growth_past_capacity_and_fallback(gpu):
    """A 40-validator state grows past its storage several times up to 5 000 validators, then one edit dirties more
    than 65 536 leaves of one tree: the root falls back to rebuilding the trees from the resident items at their
    current lengths; the next root is warm again."""
    rng = np.random.default_rng(40)
    model = StateModel(beacon_state_deneb_ssz(40, seed=4, n_votes=2, n_summaries=1), "deneb")
    st = resident(model)
    for target in (100, 350, 1200, 5000):
        apply(st, model, deposits(rng, model, target - model.length("validators")))
        check(st, model, warm="bulk")
    apply(st, model, deposits(rng, model, 70_000))
    check(st, model, warm=False, fresh=False)
    patch(st, model, "validators", 121 * 74_000 + 80, struct.pack("<Q", 7))
    apply(st, model, [("eth1_data_votes", 3, 2, rb(rng, 72))])
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
def test_electra_pending_drain_fallback(gpu):
    """A front drain of a long pending list dirties more than 65 536 leaves: fallback, then warm again."""
    rng = np.random.default_rng(41)
    model = StateModel(beacon_state_deneb_ssz(37, seed=6, fork="electra", n_pending=(70_000, 2, 2)), "electra")
    st = resident(model)
    rest = bytes(model.parts["pending_balance_deposits"][16 * 100:])
    apply(st, model, [("pending_balance_deposits", 69_900, 0, rest)])
    check(st, model, warm=False, fresh=False)
    apply(st, model, [("pending_balance_deposits", 69_901, 69_900, rb(rng, 16))])
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
def test_packed_tails(gpu):
    """Truncating a packed list whose last chunk keeps some items zeroes the rest of that chunk; growing it again
    does not bring the old bytes back."""
    rng = np.random.default_rng(12)
    model = StateModel(beacon_state_deneb_ssz(1001, seed=8), "deneb")
    st = resident(model)
    apply(st, model, [("balances", 997, 997, b""), ("inactivity_scores", 990, 990, b""),
                      ("previous_epoch_participation", 970, 970, b"")])
    check(st, model, warm=True)
    apply(st, model, [("balances", 999, 997, rb(rng, 16)), ("previous_epoch_participation", 980, 970, bytes(10))])
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["bellatrix", "capella", "deneb", "electra"])
def test_conversion_by_payload_header(gpu, fork):
    """The call that converts the handle replaces the payload header (extra_data changes length); list edits follow
    on the converted handle."""
    rng = np.random.default_rng(21)
    model = StateModel(beacon_state_deneb_ssz(300, seed=12, fork=fork), fork)
    st = resident(model)
    hdr = header_bytes(rng, fork, 7)
    st.set_payload_header(hdr)
    model.parts["latest_execution_payload_header"][:] = hdr
    check(st, model, warm=True)
    apply(st, model, deposits(rng, model, 3))
    patch(st, model, "latest_execution_payload_header", 0, rb(rng, 32))
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
def test_conversion_before_the_first_root(gpu):
    """A list edit straight after enable_incremental: the lists convert before any root has built the levels."""
    from lighthouse_b200 import tree_hash as T
    rng = np.random.default_rng(22)
    model = StateModel(beacon_state_deneb_ssz(1001, seed=13), "deneb")
    st = T.ResidentState(model.ssz(), "deneb")
    st.enable_incremental()
    apply(st, model, deposits(rng, model, 5))
    check(st, model, warm=False)
    patch(st, model, "balances", 8 * 3, struct.pack("<Q", 77))
    patch(st, model, 176 + 32 * 9, 0, rb(rng, 32))                                       # block root
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
def test_conversion_with_patches_pending(gpu):
    """Validators and balances are patched with no root in between, then the next call converts: the lists take the
    patched bytes along."""
    rng = np.random.default_rng(23)
    model = StateModel(beacon_state_deneb_ssz(20_000, seed=14, n_votes=5), "deneb")
    st = resident(model)
    for vi in rng.choice(20_000, size=50, replace=False):
        patch(st, model, "validators", 121 * int(vi) + 80, struct.pack("<Q", int(rng.integers(1, 1 << 40))))
        patch(st, model, "balances", 8 * int(vi), struct.pack("<Q", int(rng.integers(1, 1 << 40))))
    apply(st, model, [("eth1_data_votes", 6, 5, rb(rng, 72))])
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["deneb", "electra"])
def test_conversion_of_a_small_state(gpu, fork):
    """Every list has at most 8 leaves, so its stage-time field root came from small-tree ops rather than reduce
    passes; votes, summaries and the pending lists start empty."""
    rng = np.random.default_rng(24)
    model = StateModel(beacon_state_deneb_ssz(6, seed=15, fork=fork, n_votes=0, n_summaries=0, n_pending=(0, 0, 0)),
                       fork)
    st = resident(model)
    apply(st, model, deposits(rng, model, 2) + [("eth1_data_votes", 1, 0, rb(rng, 72))])
    check(st, model, warm=True)
    apply(st, model, [("historical_summaries", 1, 0, rb(rng, 64))])
    check(st, model, warm=True)
    st.release()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["capella", "electra"])
def test_patches_where_an_emptied_list_ends(gpu, fork):
    """Lists emptied by an epoch end where the next field starts: patches there still find the next field's bytes."""
    rng = np.random.default_rng(25)
    model = StateModel(beacon_state_deneb_ssz(37, seed=16, fork=fork, n_votes=5, n_summaries=3), fork)
    st = resident(model)
    empty = [("eth1_data_votes", 0, 0, b"")]
    if fork == "electra":
        empty += [(n, 0, 0, b"") for n in ("pending_balance_deposits", "pending_partial_withdrawals",
                                           "pending_consolidations")]
    apply(st, model, empty)
    apply(st, model, deposits(rng, model, 70_000))
    for name in ("validators", "balances"):
        n = model.length(name)
        for i in (0, n // 2, n - 3):
            patch(st, model, name, model.item_bytes(name) * i, rb(rng, 8))
    check(st, model, warm=False, fresh=False)
    st.release()


@pytest.mark.gpu
def test_refusals_leave_the_handle_unchanged(gpu):
    from lighthouse_b200 import Lhb200Error, _ffi, tree_hash as T
    rng = np.random.default_rng(13)
    model = StateModel(beacon_state_deneb_ssz(500, seed=10, fork="capella"), "capella")
    st = resident(model)
    apply(st, model, [("eth1_data_votes", model.length("eth1_data_votes") + 1, model.length("eth1_data_votes"),
                       rb(rng, 72))])
    before = st.root()
    nv = model.length("validators")
    cases = [
        ([(13, 1, 0, 1)], rb(rng, 32)),                                          # a vector, not a list
        ([(7, 1, 0, 1)], rb(rng, 32)),                                           # historical_roots: not resizable
        ([(99, 1, 0, 1)], rb(rng, 32)),                                          # no such field
        ([(34, 1, 0, 1)], rb(rng, 16)),                                          # a field Capella lacks
        ([(9, 2049, 0, 2049)], rb(rng, 72 * 2049)),                              # limit overrun
        ([(11, nv + 2, nv, 1)], validators_ssz(1, rng)),                         # short write on growth
        ([(12, nv, nv - 1, 2)], rb(rng, 16)),                                    # first + n > new_len
        ([(12, nv, 0, 1), (12, nv, 1, 1)], rb(rng, 16)),                         # two edits of one field
    ]
    for edits, data in cases:
        assert raw_edit(st, edits, data) == _ffi.EINVAL, edits
        assert st.root() == before
    e = (_ffi.ListEdit * 1)(_ffi.ListEdit(12, 1, nv, 0, 0))                         # reserved != 0
    assert _ffi.lib.lhb200_state_list_edit(st._h, C.cast(e, C.c_void_p), 1, None) == _ffi.EINVAL
    with pytest.raises(Lhb200Error):
        st.set_payload_header(header_bytes(rng, "capella", 33))                  # extra_data over its limit
    assert st.root() == before
    check(st, model, warm=True)
    cold = T.ResidentState(model.ssz(), "capella")                               # not incremental
    with pytest.raises(Lhb200Error) as e:
        cold.truncate("balances", 3)
    assert e.value.code == _ffi.EINVAL
    cold.release()
    deneb = beacon_state_deneb_ssz(300, seed=1)
    sh = T.ShardedState(deneb, 0, 2)                                             # sharded
    assert raw_edit(sh, [(12, 299, 299, 0)]) == _ffi.EINVAL
    sh.release()
    st.release()


def test_entry_points_need_a_device():
    """Without a device every new entry point refuses with ENODEV instead of computing anything on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    e = (_ffi.ListEdit * 1)(_ffi.ListEdit(9, 0, 0, 0, 0))
    n = C.c_uint64(0)
    assert _ffi.lib.lhb200_state_list_edit(None, C.cast(e, C.c_void_p), 1, None) == _ffi.ENODEV
    assert _ffi.lib.lhb200_state_list_len(None, 9, C.byref(n)) == _ffi.ENODEV
    assert _ffi.lib.lhb200_state_set_payload_header(None, b"\0" * 584, 584) == _ffi.ENODEV
