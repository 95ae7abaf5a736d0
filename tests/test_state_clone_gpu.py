"""BeaconState::clone of a resident handle (lhb200_state_clone): a clone has its own device memory and the source's
encoding, lengths, pending mutations and warm state, so two branches of one state root warm and independently.

Models and helpers are the ones of tests/test_state_lists_gpu.py: Deneb is checked against the C oracle, every fork
against the from-spec merkleization of tests/ssz_spec.py."""
import copy
import ctypes as C
import gc
import struct

import numpy as np
import pytest

from lighthouse_b200.synthetic import beacon_state_deneb_ssz
from tests.test_state_lists_gpu import (StateModel, apply, check, deposits, header_bytes, patch, rb, resident)

FORKS = ["altair", "bellatrix", "capella", "deneb", "electra"]


def disjoint(a, b):
    from lighthouse_b200 import _ffi
    d = C.c_int32(-1)
    assert _ffi.lib.lhb200_debug_state_disjoint(a._h, b._h, C.byref(d)) == _ffi.OK
    return d.value


def launches():
    from lighthouse_b200 import _ffi
    return _ffi.lib.lhb200_launch_count()


def vote(rng, model):
    n = model.length("eth1_data_votes")
    return [("eth1_data_votes", n + 1, n, rb(rng, 72))]


@pytest.mark.gpu
@pytest.mark.parametrize("fork", FORKS)
def test_clone_of_a_staged_handle(gpu, fork):
    """A freshly staged, non-incremental handle: the clone hashes like its source and shares no device memory."""
    from lighthouse_b200 import tree_hash as T
    gc.collect()
    model = StateModel(beacon_state_deneb_ssz(300, seed=31, fork=fork), fork)
    src = T.ResidentState(model.ssz(), fork)
    c = src.clone()
    assert c.fork == fork
    assert c.device_bytes == src.device_bytes > 0
    assert disjoint(c, src) == disjoint(src, c) == 1
    assert disjoint(src, src) == 0
    check(c, model, fresh=False)
    check(src, model)
    assert c.root(want_field_roots=True) == src.root(want_field_roots=True)
    assert c.hash_units == src.hash_units
    src.release()
    check(c, model)
    c.release()


@pytest.mark.gpu
@pytest.mark.parametrize("n_validators", [20_000, 32_760])
def test_divergent_branches(gpu, n_validators):
    """Two clones of one converted parent follow different slots, each warm; the parent stays as it was.  Branch A takes
    deposits (32 760 + 16 crosses a power of two in five trees) and balance and participation patches; branch B takes
    eth1 votes, headers whose extra_data changes length, and a participation rotation."""
    rng = np.random.default_rng(n_validators + 1)
    model = StateModel(beacon_state_deneb_ssz(n_validators, seed=17, n_votes=5, n_summaries=3), "deneb")
    parent = resident(model)
    apply(parent, model, vote(rng, model))                       # converts the parent
    check(parent, model, warm=True, fresh=False)
    before = parent.root(want_field_roots=True)
    a, b = parent.clone(), parent.clone()
    ma, mb = copy.deepcopy(model), copy.deepcopy(model)
    assert disjoint(a, b) == disjoint(a, parent) == disjoint(parent, b) == 1
    for slot in range(4):
        apply(a, ma, deposits(rng, ma, 16))
        nv = ma.length("validators")
        for vi in rng.choice(nv, size=20, replace=False):
            patch(a, ma, "balances", 8 * int(vi), struct.pack("<Q", int(rng.integers(1, 1 << 40))))
        patch(a, ma, "current_epoch_participation", int(rng.integers(0, nv - 300)),
              bytes(rng.integers(0, 8, size=300, dtype=np.uint8)))
        check(a, ma, warm=True)

        apply(b, mb, vote(rng, mb))
        hdr = header_bytes(rng, "deneb", (7 * slot + 3) % 33)
        b.set_payload_header(hdr)
        mb.parts["latest_execution_payload_header"][:] = hdr
        if slot == 2:
            nv = mb.length("validators")
            apply(b, mb, [("previous_epoch_participation", nv, 0, bytes(mb.parts["current_epoch_participation"])),
                          ("current_epoch_participation", nv, 0, bytes(nv))])
        check(b, mb, warm=True)
    assert parent.root(want_field_roots=True) == before
    assert parent.list_len("validators") == n_validators
    for h in (a, b, parent):
        h.release()


@pytest.mark.gpu
def test_clone_with_mutations_pending(gpu):
    """Patches and list edits made without a root in between travel with the clone: both handles root warm to the
    patched state.  Before the first list edit the pending patches sit in the unconverted handle's dirty bitmaps."""
    rng = np.random.default_rng(33)
    model = StateModel(beacon_state_deneb_ssz(1001, seed=18, n_votes=4), "deneb")
    parent = resident(model)
    for vi in (3, 500, 1000):
        patch(parent, model, "validators", 121 * vi + 80, struct.pack("<Q", 1000 + vi))
        patch(parent, model, "balances", 8 * vi, struct.pack("<Q", 2000 + vi))
    first = parent.clone()
    m1 = copy.deepcopy(model)
    patch(parent, model, 176 + 32 * 5, 0, rb(rng, 32))                                   # block root
    apply(parent, model, deposits(rng, model, 3) + vote(rng, model))
    patch(parent, model, "balances", 8 * 1002, struct.pack("<Q", 77))
    second = parent.clone()
    check(first, m1, warm=True)
    check(second, model, warm=True)
    check(parent, model, warm=True)
    for h in (first, second, parent):
        h.release()


@pytest.mark.gpu
def test_clone_before_conversion(gpu):
    """A clone of an incremental handle that has not converted converts on its own first list edit; the parent keeps
    patching unconverted and converts later."""
    rng = np.random.default_rng(34)
    model = StateModel(beacon_state_deneb_ssz(1001, seed=19, n_votes=2), "deneb")
    parent = resident(model)
    c = parent.clone()
    mc = copy.deepcopy(model)
    apply(c, mc, deposits(rng, mc, 5) + vote(rng, mc))
    check(c, mc, warm=True)
    patch(parent, model, "balances", 8 * 10, struct.pack("<Q", 5))
    check(parent, model, warm=True)
    apply(parent, model, [("historical_summaries", model.length("historical_summaries") + 1,
                           model.length("historical_summaries"), rb(rng, 64))])
    check(parent, model, warm=True)
    patch(c, mc, "validators", 121 * 1004 + 80, struct.pack("<Q", 9))
    check(c, mc, warm=True)
    for h in (c, parent):
        h.release()


@pytest.mark.gpu
@pytest.mark.parametrize("release_clone_first", [False, True])
def test_clone_outlives_its_source(gpu, release_clone_first):
    """The source is released and its arena goes to the next staged state; the clone then grows a list past its
    capacity, takes an edit that dirties more than 65 536 leaves, and is cloned in turn before that root."""
    from lighthouse_b200 import tree_hash as T
    rng = np.random.default_rng(35)
    model = StateModel(beacon_state_deneb_ssz(300, seed=20, n_votes=2, n_summaries=1), "deneb")
    src = resident(model)
    apply(src, model, vote(rng, model))
    c = src.clone()
    src.release()
    other_model = StateModel(beacon_state_deneb_ssz(300, seed=21), "deneb")
    other = T.ResidentState(other_model.ssz(), "deneb")                  # takes the released arena
    check(other, other_model, fresh=False)
    check(c, model, warm=True)
    apply(c, model, deposits(rng, model, 400))                           # past the 600-item storage
    check(c, model, warm="bulk")
    apply(c, model, deposits(rng, model, 70_000))                        # > 65 536 dirty leaves
    d = c.clone()
    md = copy.deepcopy(model)
    check(c, model, warm=False, fresh=False)
    check(d, md, warm=False, fresh=False)
    first, second, m_second = (c, d, md) if release_clone_first else (d, c, model)
    first.release()
    apply(second, m_second, vote(rng, m_second))
    patch(second, m_second, "balances", 8 * 70_500, struct.pack("<Q", 3))
    check(second, m_second, warm=True)
    check(other, other_model, fresh=False)
    second.release()
    other.release()


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["capella", "electra", "altair"])
def test_clone_round_other_forks(gpu, fork):
    rng = np.random.default_rng(36)
    model = StateModel(beacon_state_deneb_ssz(300, seed=22, fork=fork), fork)
    parent = resident(model)
    apply(parent, model, deposits(rng, model, 2))
    want = parent.root(want_field_roots=True)
    c = parent.clone()
    mc = copy.deepcopy(model)
    apply(c, mc, deposits(rng, mc, 16) + vote(rng, mc))
    patch(c, mc, "balances", 8 * 7, struct.pack("<Q", 99))
    if fork != "altair":
        hdr = header_bytes(rng, fork, 5)
        c.set_payload_header(hdr)
        mc.parts["latest_execution_payload_header"][:] = hdr
    check(c, mc, warm=True)
    assert parent.root(want_field_roots=True) == want
    check(parent, model, warm=True)
    for h in (c, parent):
        h.release()


@pytest.mark.gpu
def test_clone_is_one_launch(gpu):
    """All live bytes of a converted handle move in one k_copy_ranges launch."""
    from lighthouse_b200 import _ffi
    rng = np.random.default_rng(37)
    model = StateModel(beacon_state_deneb_ssz(20_000, seed=23), "deneb")
    parent = resident(model)
    apply(parent, model, deposits(rng, model, 4))
    parent.root()
    n0 = launches()
    c = parent.clone()
    assert launches() - n0 == 1
    assert c.device_bytes == parent.device_bytes
    live = C.c_uint64(0)
    assert _ffi.lib.lhb200_debug_state_live_bytes(parent._h, C.byref(live)) == _ffi.OK
    assert 0 < live.value < parent.device_bytes
    check(c, model, warm=True, fresh=False)
    for h in (c, parent):
        h.release()


@pytest.mark.gpu
def test_clone_refusals(gpu):
    from lighthouse_b200 import _ffi, tree_hash as T
    lib = _ffi.lib
    deneb = beacon_state_deneb_ssz(300, seed=1)
    sh = T.ShardedState(deneb, 0, 2)
    sentinel = C.c_void_p(0x1234)
    assert lib.lhb200_state_clone(sh._h, C.byref(sentinel)) == _ffi.EINVAL
    assert sentinel.value == 0x1234
    sh.release()
    st = T.ResidentState(deneb, "deneb")
    n, d = C.c_uint64(0), C.c_int32(-1)
    assert lib.lhb200_state_clone(None, C.byref(sentinel)) == _ffi.EINVAL
    assert lib.lhb200_state_clone(st._h, None) == _ffi.EINVAL
    assert sentinel.value == 0x1234
    assert lib.lhb200_state_device_bytes(None, C.byref(n)) == _ffi.EINVAL
    assert lib.lhb200_state_device_bytes(st._h, None) == _ffi.EINVAL
    assert lib.lhb200_debug_state_disjoint(None, st._h, C.byref(d)) == _ffi.EINVAL
    assert lib.lhb200_debug_state_disjoint(st._h, None, C.byref(d)) == _ffi.EINVAL
    assert lib.lhb200_debug_state_disjoint(st._h, st._h, None) == _ffi.EINVAL
    st.release()
