"""Phase0 (Base) BeaconStates and BeaconBlocks on the device: the mainnet and Sepolia genesis states and the mainnet
genesis block against their golden roots, synthetic states and blocks against the from-spec merkleization, malformed
input, and a warm replay whose blocks append pending attestations and whose epoch rotates them, with a clone."""
import ctypes as C
import struct

import numpy as np
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic
from tests import ssz_proof_spec, ssz_spec
from tests.phase0_state import (BASE, O_BLOCK_ROOTS, O_PP_OFF, O_SLOT, O_STATE_ROOTS, Chain, SpecRoots, genesis_block,
                                genesis_state, join_fields, split_fields, with_pending)
from tests.test_ssz_layouts_gpu import malformed

pytestmark = pytest.mark.gpu


def _einval(fn):
    from lighthouse_b200 import Lhb200Error
    from lighthouse_b200._ffi import EINVAL
    with pytest.raises(Lhb200Error) as e:
        fn()
    assert e.value.code == EINVAL, e.value


def verify(leaf, branch, gindex, root):
    assert len(branch) == gindex.bit_length() - 1
    assert ssz_proof_spec.root_from_branch(leaf, branch, gindex) == root, gindex


# ---- genesis pins ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["mainnet", "sepolia"])
def test_gpu_genesis_state_roots(gpu, net):
    from lighthouse_b200 import tree_hash as T
    ssz, meta = genesis_state(net)
    want = bytes.fromhex(meta["state_root"])
    want_fields = SpecRoots().fields(ssz)
    root, fields = T.beacon_state_root(ssz, "base", want_field_roots=True)
    assert root == want
    assert fields[:21] == want_fields and fields[21:] == [bytes(32)] * 7
    st = T.ResidentState(ssz, "base")
    try:
        assert st.root() == want
        g = list(range(32, 53))   # the 21 field roots below the 32-leaf top tree
        r, branches = st.proofs(g)
        assert r == want
        for gi, br, leaf in zip(g, branches, want_fields):
            verify(leaf, br, gi, want)
        st.enable_incremental()
        assert st.root() == want and st.root() == want
    finally:
        st.release()


def test_gpu_mainnet_genesis_block_root(gpu):
    from lighthouse_b200 import tree_hash as T
    _, meta = genesis_state("mainnet")
    block = S.serialize(S.BeaconBlockBase, genesis_block(bytes.fromhex(meta["state_root"])))
    assert T.beacon_block_roots([block], "base")[0].hex() == meta["genesis_block_root"] == \
        "4d611d5b93fdab69013a7f0a2f961caca0c853f87cfe9595fe50038163079360"


# ---- synthetic states -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_val,lens", [(0, (0, 0)), (40, (1, 4096)), (20000, (4096, 4096))])
def test_gpu_synthetic_base_states(gpu, n_val, lens):
    from lighthouse_b200 import tree_hash as T
    ssz = synthetic.beacon_state_deneb_ssz(n_val, seed=n_val + 3, fork="base", n_hist_roots=5, n_votes=7,
                                           n_pending_attestations=lens)
    want, want_fields = SpecRoots().root(ssz)
    root, fields = T.beacon_state_root(ssz, "base", want_field_roots=True)
    assert fields[:21] == want_fields and root == want
    st = T.ResidentState(ssz, "base")
    try:
        assert st.root() == want
        assert [st.list_len(15), st.list_len(16)] == list(lens)
    finally:
        st.release()


# ---- malformed input ------------------------------------------------------------------------------------------------
def _expect_einval_all(fn, cases):
    from lighthouse_b200 import Lhb200Error
    from lighthouse_b200._ffi import EINVAL
    accepted = []
    for label, b in cases:
        try:
            fn(b)
            accepted.append(label)
        except Lhb200Error as e:
            assert e.code == EINVAL, (label, e)
    assert not accepted, accepted


def _pending_cases(rng):
    """(label, list SSZ) of malformed pending-attestation lists."""
    good = [synthetic.pending_attestation_ssz(rng, 12) for _ in range(3)]
    too_many_bits = synthetic.pending_attestation_ssz(rng, 2049)
    no_delim = good[1][:-1] + b"\0"
    return [("2049 bits", synthetic.pending_attestations_list_ssz(good[:1] + [too_many_bits])),
            ("missing delimiter", synthetic.pending_attestations_list_ssz([good[0], no_delim, good[2]])),
            ("4097 records", synthetic.pending_attestations_list_ssz(good[:1] * 4097)),
            ("record below its fixed part", synthetic.pending_attestations_list_ssz([good[0], good[1][:148]])),
            ("bitlist offset not 148", synthetic.pending_attestations_list_ssz([good[0], b"\x95\0\0\0" + good[1][4:]]))]


def test_gpu_malformed_base_states_and_blocks(gpu):
    from lighthouse_b200 import tree_hash as T
    ssz = synthetic.beacon_state_deneb_ssz(40, seed=91, fork="base", n_hist_roots=3, n_votes=2,
                                           n_pending_attestations=(2, 2), pending_bit_lengths=(5, 300))
    assert T.beacon_state_root(ssz, "base") == SpecRoots().root(ssz)[0]
    cases = malformed(BASE, ssz)
    labels = " ".join(label for label, _ in cases)
    assert "aggregation_bits: one over the limit" in labels, labels
    rng = np.random.default_rng(5)
    ok = synthetic.pending_attestations_list_ssz([synthetic.pending_attestation_ssz(rng, 7)])
    cases += [(label, with_pending(ssz, ok, b)) for label, b in _pending_cases(rng)]
    cases += [(label + " (previous)", with_pending(ssz, b, ok)) for label, b in _pending_cases(rng)]
    _expect_einval_all(lambda b: T.beacon_state_root(b, "base"), cases)
    value, blk = synthetic.beacon_block_deneb(seed=90, fork="base", n_attestations=2, committee=20, n_exits=1)
    assert T.beacon_block_roots([blk], "base") == [ssz_spec.hash_tree_root(S.BeaconBlockBase, value)]
    bcases = malformed(S.BeaconBlockBase, blk)
    assert len(bcases) > 30, len(bcases)
    _expect_einval_all(lambda b: T.beacon_block_roots([b], "base"), bcases)


# ---- blocks ---------------------------------------------------------------------------------------------------------
def test_gpu_base_blocks(gpu):
    from lighthouse_b200 import tree_hash as T
    blocks = []
    for i, n_att in enumerate([0, 1, 128]):
        value, blk = synthetic.beacon_block_deneb(seed=40 + i, fork="base", n_attestations=n_att, n_proposer_slashings=1,
                                                  n_attester_slashings=1, n_deposits=2, n_exits=3)
        blocks.append((value, blk))
        want = ssz_spec.hash_tree_root(S.BeaconBlockBase, value)
        roots, bodies = T.beacon_block_roots([blk], "base", want_body_roots=True)
        assert roots == [want] and bodies == [ssz_spec.hash_tree_root(S.BeaconBlockBodyBase, value["body"])]
        # a Base block hashed as Altair: refused, or another root
        try:
            assert T.beacon_block_roots([blk], "altair") != [want]
        except Exception as e:
            from lighthouse_b200._ffi import EINVAL
            assert getattr(e, "code", None) == EINVAL, e
    _einval(lambda: T.beacon_block_roots([blocks[0][1]], "base", blinded=True))
    batch = [synthetic.beacon_block_deneb(seed=60 + i, fork="base", n_attestations=i * 4, committee=100 + i)
             for i in range(32)]
    assert T.beacon_block_roots([b for _, b in batch], "base") == \
        [ssz_spec.hash_tree_root(S.BeaconBlockBase, v) for v, _ in batch]
    # every body field gindex (8 fields: a 8-leaf body tree) in every block, and a record root below attestations
    value, blk = blocks[2]
    g = list(range(8, 16)) + [(13 * 2) * 128 + 5]
    body_roots, branches = T.beacon_block_body_proofs([blk], [(0, x) for x in g], "base")
    body_root = ssz_spec.hash_tree_root(S.BeaconBlockBodyBase, value["body"])
    assert body_roots == [body_root]
    leaves = [ssz_spec.hash_tree_root(ft, value["body"][n]) for n, ft in S.BeaconBlockBodyBase[1]]
    leaves.append(ssz_spec.hash_tree_root(S.Attestation, value["body"]["attestations"][5]))
    for gi, br, leaf in zip(g, branches, leaves):
        verify(leaf, br, gi, body_root)


# ---- resident handles: warm replay, clone, refusals, launch count ---------------------------------------------------
def _slot(st, chain, spec, slot, rng, n_att=128):
    """One block: slot, block and state roots, balances patched; the block's attestations appended to the current
    list; at an epoch boundary the lists rotate first (two calls)."""
    lst = synthetic.pending_attestations_list_ssz
    if slot % 32 == 0:
        chain.prev, chain.cur = chain.cur, []
        st.set_pending_attestations("previous_epoch_attestations", lst(chain.prev))
        st.set_pending_attestations("current_epoch_attestations", b"")
    edits = [(O_SLOT, struct.pack("<Q", slot)), (O_BLOCK_ROOTS + 32 * (slot % 8192), rng.bytes(32)),
             (O_STATE_ROOTS + 32 * (slot % 8192), rng.bytes(32))]
    o_bal = chain.balances_offset()
    for i in rng.choice(len(chain.f[12]) // 8, size=16, replace=False):
        edits.append((o_bal + 8 * int(i), struct.pack("<Q", int(rng.integers(0, 1 << 40)))))
    chain.patch(edits)
    st.patch_batch(edits)
    new = [synthetic.pending_attestation_ssz(rng, int(rng.choice([9, 10, 11, 300])), slot) for _ in range(n_att)]
    chain.cur = chain.cur + new
    st.set_pending_attestations(16, lst(chain.cur))
    assert st.list_len(16) == len(chain.cur) and st.list_len(15) == len(chain.prev)
    want, _ = spec.root(chain.full())
    assert st.root() == want, slot
    return want


def test_gpu_warm_replay_across_an_epoch_with_a_clone(gpu):
    from lighthouse_b200 import tree_hash as T
    start = 32 * 100 + 20
    ssz = synthetic.beacon_state_deneb_ssz(20000, seed=17, fork="base", n_hist_roots=2, n_votes=3,
                                           n_pending_attestations=(4000, 20 * 128), pending_bit_lengths=(10, 11, 300))
    ssz = bytearray(ssz)
    struct.pack_into("<Q", ssz, O_SLOT, start - 1)
    spec = SpecRoots()
    chain = Chain(bytes(ssz))
    st = T.ResidentState(bytes(ssz), "base")
    clone = None
    try:
        assert st.root() == spec.root(chain.full())[0]
        st.enable_incremental()
        rng = np.random.default_rng(1)
        for k in range(40):
            _slot(st, chain, spec, start + k, rng)
            if k == 8:   # a branch: the clone takes other blocks, then both go on
                clone, cchain = st.clone(), Chain(chain.full())
                crng = np.random.default_rng(2)
            if clone is not None and k < 16:
                want = _slot(clone, cchain, spec, start + k + 1, crng, n_att=64)
                # record-level proofs on the clone: previous and current lists, first / last records
                g = [48 * 2 * 4096 + 0, 48 * 2 * 4096 + len(cchain.cur) - 1, 47 * 2 * 4096 + 3]
                r, branches = clone.proofs(g)
                assert r == want
                leaves = [spec.record_root(cchain.cur[0]), spec.record_root(cchain.cur[-1]),
                          spec.record_root(cchain.prev[3])]
                for gi, br, leaf in zip(g, branches, leaves):
                    verify(leaf, br, gi, want)
                _einval(lambda: clone.proofs([48 * 2 * 4096 * 2]))   # below a record root
            if clone is not None and k == 15:
                clone.release()
                clone = None
        assert st.root() == spec.root(chain.full())[0]
    finally:
        st.release()
        if clone is not None:
            clone.release()


def test_gpu_pending_refusals_leave_the_root(gpu):
    from lighthouse_b200 import _ffi, tree_hash as T
    ssz = synthetic.beacon_state_deneb_ssz(300, seed=23, fork="base", n_pending_attestations=(5, 6))
    want = SpecRoots().root(ssz)[0]
    rng = np.random.default_rng(3)
    ok = synthetic.pending_attestations_list_ssz([synthetic.pending_attestation_ssz(rng, 7)])
    st = T.ResidentState(ssz, "base")
    deneb = T.ResidentState(synthetic.beacon_state_deneb_ssz(40, seed=2), "deneb")
    try:
        _einval(lambda: st.set_pending_attestations(15, ok))        # not incremental
        assert st.root() == want
        st.enable_incremental()
        deneb.enable_incremental()
        _einval(lambda: deneb.set_pending_attestations(15, ok))     # not a Base handle
        for field in (14, 17, 21):
            _einval(lambda: st.set_pending_attestations(field, ok))
        for label, b in _pending_cases(rng):
            _einval(lambda: st.set_pending_attestations(16, b))
        for field in (15, 16, 21):
            edit = (_ffi.ListEdit * 1)(_ffi.ListEdit(field, 0, 0, 0, 0))
            assert _ffi.lib.lhb200_state_list_edit(st._h, C.cast(edit, C.c_void_p), 1, None) == _ffi.EINVAL
        assert st.root() == want
        # list_edit of fields 9 / 11 / 12 goes on working, and moves the pending lists' offsets along
        f = split_fields(ssz)
        st.append("balances", struct.pack("<Q", 5))
        st.set_pending_attestations(15, ok)
        f[12] += struct.pack("<Q", 5)
        f[15] = ok
        want2 = SpecRoots().root(join_fields(f))[0]
        assert st.root() == want2
        # patches that reach a pending list are refused and change nothing, in the same batch as a valid patch too:
        # its offset table and bitlists steer the device reads, and change only through set_pending_attestations
        full = join_fields(f)
        o_pp, o_cp = struct.unpack_from("<II", full, O_PP_OFF)
        first = struct.unpack_from("<I", f[16], 0)[0]
        for off, b in [(o_cp, b"\xff\xff\xff\x7f"),               # the first record's offset
                       (o_cp + first, b"\0\0\0\0"),                 # its bitlist offset
                       (o_cp + first + 30, b"\x7e"),                   # its beacon_block_root
                       (len(full) - 1, b"\0"),                         # the last bitlist's delimiter
                       (o_pp + len(ok) - 2, b"\x01\x00"),             # across the end of the previous list
                       (o_pp - 1, b"\0\0")]:                            # the last balance byte and the list
            _einval(lambda: st.patch(off, b))
            _einval(lambda: st.patch_batch([(O_SLOT, b"\x01"), (off, b)]))
        assert st.root() == want2
        st.patch(O_SLOT, b"\x01")   # the fixed fields still patch
        f[2] = b"\x01" + f[2][1:]
        want2 = SpecRoots().root(join_fields(f))[0]
        assert st.root() == want2
        # hash units follow the current record counts
        u0 = st.hash_units
        st.set_pending_attestations(16, synthetic.pending_attestations_list_ssz(
            [synthetic.pending_attestation_ssz(rng, 9) for _ in range(40)]))
        assert st.hash_units - u0 == 19 * (40 - 6)
        st.set_pending_attestations(16, f[16])
        assert st.hash_units == u0 and st.root() == want2
        _einval(lambda: st.set_pending_attestations(15, ok[:-1]))
        assert st.root() == want2
    finally:
        st.release()
        deneb.release()


def test_gpu_pending_lists_rerooted_by_one_launch(gpu):
    from lighthouse_b200 import tree_hash as T
    from lighthouse_b200._ffi import lib
    ssz = synthetic.beacon_state_deneb_ssz(1000, seed=29, fork="base", n_pending_attestations=(50, 60))
    rng = np.random.default_rng(4)
    lst = synthetic.pending_attestations_list_ssz
    st = T.ResidentState(ssz, "base")
    try:
        st.enable_incremental()
        st.root()
        st.set_pending_attestations(15, lst([synthetic.pending_attestation_ssz(rng, 20) for _ in range(70)]))
        st.root()
        n0 = lib.lhb200_launch_count()
        st.set_pending_attestations(16, lst([synthetic.pending_attestation_ssz(rng, 20) for _ in range(10)]))
        st.root()
        one = lib.lhb200_launch_count() - n0
        n0 = lib.lhb200_launch_count()
        st.set_pending_attestations(15, lst([synthetic.pending_attestation_ssz(rng, 30) for _ in range(90)]))
        st.set_pending_attestations(16, lst([synthetic.pending_attestation_ssz(rng, 30) for _ in range(80)]))
        import torch
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            st.root()
            torch.cuda.synchronize()
        both = lib.lhb200_launch_count() - n0
        assert both == one, (both, one)
        names = [e.name for e in prof.events() if "pending_attestation_roots" in e.name]
        assert len(names) == 1, names
    finally:
        st.release()
