"""lhb200_attestations_verify and device-resident committee caches against the restatement of
tests/attestation_spec.py (committees from tests/committee_spec.py): indices and signing roots for Base, Deneb and
Electra attestations at 1 to 500 000 validators with caches of three epochs and both sides of the fork epoch; the
verdicts with bad signatures, flipped bits and every indexing error; bit-exactness with Batch.upload_indexed over the
restatement's sets; grouping; handle lifetime; concurrent callers; launch counts; refusals.  The test without a device
runs in the CPU suite."""
import ctypes as C
import threading

import numpy as np
import pytest

from lighthouse_b200.synthetic import (MAINNET_GVR, attestation_data_ssz, attestation_ssz, beacon_state_deneb_ssz,
                                       interop_secret_keys, signed_attestations)
from tests import attestation_spec as A
from tests import committee_spec as CS

EPOCH = 100
GVR = MAINNET_GVR
V_PREV, V_CUR = bytes.fromhex("03000000"), bytes.fromhex("04000000")
FORK_AT_CURRENT = (V_PREV, V_CUR, EPOCH)   # the previous epoch signs with the previous version, the others the current
_worlds, _sks = {}, {}


class World:
    """A resident state of n validators at EPOCH, its host caches (restatement) and device caches for EPOCH - 1 ..
    EPOCH + 1, and a pubkey table of the n interop keys."""

    def __init__(self, n, fork):
        from lighthouse_b200 import bls, tree_hash as T
        from lighthouse_b200.synthetic import interop_pubkey_table
        ssz = bytearray(beacon_state_deneb_ssz(n, seed=5, fork=fork, n_votes=3, n_hist_roots=5, n_summaries=2))
        CS.set_slot(ssz, EPOCH * 32 + 9)
        self.ssz, self.fork, self.n = bytes(ssz), fork, n
        self.state = T.ResidentState(self.ssz, fork)
        s = CS.State(self.ssz)
        self.epochs = (EPOCH - 1, EPOCH, EPOCH + 1)
        self.host = [CS.committee_cache(s, e) for e in self.epochs]
        self.dev = [self.state.device_committee_cache(e) for e in self.epochs]
        if n not in _sks:   # shared by the forks' worlds of one size
            _sks[n] = interop_secret_keys(n)
        self.sks = _sks[n]
        self.table = bls.PubkeyTable(n)
        self.table.append(interop_pubkey_table(n).tobytes())

    def host_cache(self, e):
        from lighthouse_b200.committees import CommitteeCache
        c = self.host[self.epochs.index(e)]
        return CommitteeCache(c["epoch"], c["shuffling"], c["positions"], c["committees_per_slot"], c["seed"])


def world(n, fork):
    key = (n, fork)
    if key not in _worlds:
        _worlds[key] = World(n, fork)
    return _worlds[key]


def run(w, atts, electra, fork_info=FORK_AT_CURRENT, rands=None, caches=None, host=None, table_len=None):
    """The call with indexed output, every output checked against the restatement -> (ok, statuses, the statuses a
    batch of valid signatures gives: the indexing codes, 4 for an empty index set, else 0)."""
    from lighthouse_b200 import attestations as AT
    caches = w.dev if caches is None else caches
    host = w.host if host is None else host
    ok, st, roots, idx = AT.verify_attestations(atts, "electra" if electra else w.fork, caches, w.table, fork_info,
                                                GVR, rands, want_indices=True)
    tl = w.n if table_len is None else table_len
    want = []
    for i, a in enumerate(atts):
        s, ind, root = A.index_attestation(a, electra, host, tl, fork_info, GVR)
        assert roots[i] == root, i
        if s in (A.OK, A.UNKNOWN_VALIDATOR):
            assert idx[i].tolist() == ind.tolist(), i
        else:
            assert len(idx[i]) == 0, i
        if s != A.OK:
            assert st[i] == s, (i, st[i], s)
        want.append(4 if s == A.OK and len(ind) == 0 else s)
    return ok, st, want


def first_slot_with_members(w, e):
    c = w.host[w.epochs.index(e)]
    return next(slot for slot, index, m in CS.committees(c) if index == 0 and len(m))


def batch(w, electra, per_epoch_kinds, fork_info=FORK_AT_CURRENT, seed=0):
    """Signed attestations over the three epochs' caches: per epoch, the (kind, n, knobs) of per_epoch_kinds."""
    out = []
    for k, e in enumerate(w.epochs):
        hc = w.host_cache(e)
        for kind, n, kw in per_epoch_kinds:
            if kind == "unaggregated":
                kw = dict(kw, slot=first_slot_with_members(w, e))
            out += signed_attestations(hc, kind, n, w.sks, fork_info, GVR, seed=seed + 97 * k, **kw)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["base", "deneb", "electra"])
@pytest.mark.parametrize("n", [1, 2048, 20_000, 500_000])
def test_indices_roots_and_verdicts(gpu, fork, n):
    w = world(n, "electra" if fork == "electra" else fork)
    electra = fork == "electra"
    if electra:
        kinds = [("electra", 4, dict(committees_per_attestation=1)), ("electra", 4, dict(committees_per_attestation=4)),
                 ("electra", 2, dict(committees_per_attestation=64, fill=0.7))]
    else:
        kinds = [("unaggregated", 64 if n > 1 else 2, dict(n_committees=2)), ("aggregate", 128 if n > 1 else 4, {})]
    for fork_info in (FORK_AT_CURRENT, (V_PREV, V_CUR, EPOCH + 2), (V_PREV, V_CUR, 0)):
        atts = batch(w, electra, kinds, fork_info)
        ok, st, want = run(w, atts, electra, fork_info)
        assert st.tolist() == want and ok == (not any(want)), st
        if n > 1:
            assert ok
    # signatures over the other fork version's domain fail
    atts = batch(w, electra, kinds, (V_PREV, V_CUR, EPOCH + 2))
    assert not run(w, atts, electra, FORK_AT_CURRENT)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["deneb", "electra"])
def test_bad_signature_flipped_bit_and_each_indexing_error(gpu, fork):
    w = world(20_000, fork)
    electra = fork == "electra"
    kinds = [("electra", 6, dict(committees_per_attestation=3, fill=0.5))] if electra else \
        [("aggregate", 12, dict(fill=0.5)), ("unaggregated", 8, dict(n_committees=2))]
    atts = batch(w, electra, kinds)
    assert run(w, atts, electra)[0]
    # one flipped signature: the batch fails, every status stays 0
    bad = list(atts)
    j = len(bad) // 2
    bad[j] = bad[j][:132] + atts[j + 1][132:228] + bad[j][228:]
    ok, st, _ = run(w, bad, electra)
    assert not ok and not st.any()
    # one flipped aggregation bit (the first byte of a bitlist of more than 8 bits: the length stays)
    bad = list(atts)
    r = bytearray(bad[3])
    fixed = A.FIXED[electra]
    assert len(r) > fixed + 1
    r[fixed] ^= 1
    bad[3] = bytes(r)
    ok, st, _ = run(w, bad, electra)
    assert not ok and not st.any()
    # each indexing error once: the others still verify, and the erroneous ones report their codes
    c = w.host[1]
    slot = EPOCH * 32 + 3
    data = attestation_data_ssz(slot, 0, bytes(32), (EPOCH - 1, bytes(32)), (EPOCH, bytes(32)))
    members = A.committee(A.spec_cache(c), slot, 0)
    full = np.ones(len(members), dtype=np.uint8)
    cb = 1 if electra else None
    far = attestation_data_ssz(slot + 64, 0, bytes(32), (EPOCH, bytes(32)), (EPOCH + 2, bytes(32)))
    no_comm = attestation_data_ssz(slot, 0 if electra else 63, bytes(32), (EPOCH - 1, bytes(32)), (EPOCH, bytes(32)))
    errs = [atts[0][:-1] + b"\x00",                                            # MALFORMED: no delimiter
            attestation_ssz(full, far, bytes(96), cb),                         # NO_CACHE
            attestation_ssz(full, no_comm, bytes(96), (1 << 63) if electra else None),   # NO_COMMITTEE
            attestation_ssz(full[:-1], data, bytes(96), cb)]                   # BITFIELD_LENGTH
    mixed = atts[:2] + errs + atts[2:]
    ok, st, _ = run(w, mixed, electra)
    assert ok and st[2:6].tolist() == [10, 11, 12, 13] and not st[:2].any() and not st[6:].any()
    # UNKNOWN_VALIDATOR: a table that stops below one attester
    from lighthouse_b200 import bls
    short = bls.PubkeyTable(w.n)
    members_of = [A.index_attestation(a, electra, w.host, w.n, FORK_AT_CURRENT, GVR)[1] for a in atts]
    cut = int(max(m.max() for m in members_of if len(m)))
    from lighthouse_b200.synthetic import interop_pubkey_table
    short.append(interop_pubkey_table(cut).tobytes())
    saved, w.table = w.table, short
    try:
        ok, st, _ = run(w, atts, electra, table_len=cut)
    finally:
        w.table = saved
        short.destroy()
    assert ok and (st == 14).sum() >= 1 and set(st.tolist()) <= {0, 14}
    # an Electra attestation without committee bits reaches the batch as a set with no keys: status 4
    if electra:
        ok, st, _ = run(w, atts[:3] + [attestation_ssz([], data, atts[0][132:228], 0)], electra)
        assert not ok and st.tolist() == [0, 0, 0, 4]


def host_route(w, atts, rands, electra=False):
    """The same sets through Batch.upload_indexed, built by the restatement -> (ok, statuses, gt, plan, launches)."""
    from lighthouse_b200 import bls
    sigs, msgs, idx, offs = b"", b"", [], [0]
    for a in atts:
        s, ind, root = A.index_attestation(a, electra, w.host, w.n, FORK_AT_CURRENT, GVR)
        assert s == A.OK
        sigs += a[132:228]
        msgs += root
        idx += ind.tolist()
        offs.append(len(idx))
    b = bls.Batch(len(atts), 1)
    b.upload_indexed(w.table, sigs, msgs, idx, offs, rands)
    b.enqueue()
    ok, st = b.result(want_status=True)
    out = ok, st, b.gt_bytes(), b.plan(), b.launches
    b.destroy()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("grouped", [False, True])
def test_bit_exact_with_upload_indexed(gpu, grouped):
    """The same sets through Batch.upload_indexed, built by the restatement, with the same scalars: the same verdict,
    statuses, kernel plan and final-exponentiated product (a swapped signature: every status 0, the pairing check
    fails, so the product is not the identity), and the same statuses with an empty signature (status 1).  The
    unaggregated batch of 64 over 2 committees runs k_g1_group_sum."""
    from lighthouse_b200 import attestations as AT
    w = world(20_000, "deneb")
    kinds = [("unaggregated", 64, dict(n_committees=2))] if grouped else [("aggregate", 40, dict(fill=0.8))]
    atts = signed_attestations(w.host_cache(EPOCH), kinds[0][0], kinds[0][1], w.sks, FORK_AT_CURRENT, GVR,
                               slot=first_slot_with_members(w, EPOCH) if grouped else None, **kinds[0][2])
    rands = np.random.default_rng(9).integers(1, 1 << 63, len(atts), dtype=np.uint64)
    swapped = list(atts)
    swapped[5] = atts[5][:132] + atts[-1][132:228] + atts[5][228:]
    empty = list(atts)
    empty[5] = atts[5][:132] + bytes(96) + atts[5][228:]
    for batch_, want_st in ((atts, 0), (swapped, 0), (empty, 1)):
        ok, st, _ = run(w, batch_, False, rands=rands)
        gt, plan = AT.last_batch_check()
        assert plan["group_sum"] == ("k_g1_group_sum" if grouped else "")
        ok2, st2, gt2, plan2, _ = host_route(w, batch_, rands)
        assert ok == ok2 == (batch_ is atts) and st.tolist() == st2.tolist() and st[5] == want_st
        assert plan == plan2
        if batch_ is not empty:   # (a batch with a failed set leaves the product unwritten)
            assert gt == gt2


@pytest.mark.gpu
def test_device_cache_lifetime(gpu):
    """A device cache equals ResidentState.committee_cache(epoch) and survives release, patch and clone of its source."""
    from lighthouse_b200 import tree_hash as T
    ssz = bytearray(beacon_state_deneb_ssz(6000, seed=8, n_votes=3, n_hist_roots=5, n_summaries=2))
    CS.set_slot(ssz, 40 * 32 + 1)
    CS.vary_validators(ssz, 40, np.random.default_rng(3))
    h = T.ResidentState(bytes(ssz), "deneb")
    want = [h.committee_cache(e) for e in (39, 40, 41)]
    dev = [h.device_committee_cache(e) for e in (39, 40, 41)]

    def same():
        for d, c in zip(dev, want):
            got = d.to_host()
            assert np.array_equal(got.shuffling(), c.shuffling()) and np.array_equal(got._positions, c._positions)
            assert got.committees_per_slot() == c.committees_per_slot() and got.seed == c.seed
            assert d.info.n_validators == 6000 and d.epoch == c.initialized_epoch
    same()
    h.patch(CS.O_RANDAO + 32 * ((40 + 65534) % 65536), bytes(32))   # the mix the current epoch's seed reads
    assert h.committee_cache(40).seed != want[1].seed
    same()
    clone = h.clone()
    h.release()
    same()
    clone.release()
    same()
    for d in dev:
        d.release()


@pytest.mark.gpu
def test_concurrent_callers_get_their_own_results(gpu):
    w = world(20_000, "deneb")
    from lighthouse_b200 import attestations as AT
    jobs = []
    for t in range(8):
        atts = batch(w, False, [("unaggregated", 8, dict(n_committees=2)), ("aggregate", 6, {})], seed=t)
        if t % 3 == 1:   # some callers carry a bad signature
            atts[4] = atts[4][:132] + atts[5][132:228] + atts[4][228:]
        jobs.append(atts)
    alone = [AT.verify_attestations(a, "deneb", w.dev, w.table, FORK_AT_CURRENT, GVR, want_indices=True) for a in jobs]
    got = [None] * 8

    def call(k):
        got[k] = AT.verify_attestations(jobs[k], "deneb", w.dev, w.table, FORK_AT_CURRENT, GVR, want_indices=True)
    threads = [threading.Thread(target=call, args=(k,)) for k in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for a, g in zip(alone, got):
        assert a[0] == g[0] and a[1].tolist() == g[1].tolist() and a[2] == g[2]
        assert [x.tolist() for x in a[3]] == [x.tolist() for x in g[3]]
    assert [a[0] for a in alone] == [t % 3 != 1 for t in range(8)]


@pytest.mark.gpu
@pytest.mark.parametrize("fork", ["deneb", "electra"])
def test_launch_count_does_not_depend_on_n(gpu, fork):
    """The call launches its two indexing kernels (and, for Electra's indexed output, one segmented sort, counted
    once) plus what verify_enqueue launches for the same sets, at 64 and at 4 096 attestations alike."""
    from lighthouse_b200 import _ffi, attestations as AT
    w = world(500_000, fork)
    electra = fork == "electra"
    kind, kw = ("electra", dict(committees_per_attestation=2)) if electra else ("aggregate", {})
    for n_att in (64, 4096):
        atts = signed_attestations(w.host_cache(EPOCH), kind, n_att, w.sks, FORK_AT_CURRENT, GVR, **kw)
        verify = host_route(w, atts, None, electra)[4]
        for want_indices in (False, True):
            AT.verify_attestations(atts, fork, w.dev, w.table, FORK_AT_CURRENT, GVR, want_indices=want_indices)
            l0 = _ffi.lib.lhb200_launch_count()
            AT.verify_attestations(atts, fork, w.dev, w.table, FORK_AT_CURRENT, GVR, want_indices=want_indices)
            got = _ffi.lib.lhb200_launch_count() - l0
            assert got == 2 + (electra and want_indices) + verify, (n_att, want_indices, got, verify)


@pytest.mark.gpu
def test_refusals_and_compute_domain(gpu):
    from lighthouse_b200 import _ffi, attestations as AT, tree_hash as T
    w = world(2048, "deneb")
    assert T.compute_domain(1, V_CUR, GVR) == A.compute_domain(1, V_CUR, GVR)
    atts = batch(w, False, [("aggregate", 3, {})])
    fid = 4

    def call(atts_, caches, fork=fid, rands=None, offs=None, cap=None):
        n = len(atts_)
        o = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum([len(a) for a in atts_], out=o[1:])
        if offs is not None:
            o = offs
        ssz = b"".join(atts_) or b"\0"
        hs = (C.c_void_p * max(len(caches), 1))(*[c._h for c in caches])
        ok = C.c_uint8()
        st = np.zeros(max(n, 1), dtype=np.uint8)
        io = np.zeros(n + 1, dtype=np.uint64)
        ix = np.zeros(1 << 16, dtype=np.uint64)
        f = AT.fork_struct(FORK_AT_CURRENT)
        return _ffi.lib.lhb200_attestations_verify(ssz, o.ctypes.data, n, fork, C.cast(hs, C.c_void_p), len(caches),
                                                   w.table._h, C.byref(f), GVR,
                                                   None if rands is None else rands.ctypes.data, C.byref(ok),
                                                   st.ctypes.data, None, io.ctypes.data if cap is not None else None,
                                                   ix.ctypes.data if cap is not None else None, cap or 0)
    assert call(atts, w.dev) == _ffi.OK
    for args, msg in (((atts[:0], w.dev), b"no attestations"), ((atts, []), b"committee caches"),
                      ((atts, w.dev + w.dev[:1]), b"committee caches"), ((atts, w.dev[:1] * 2), b"two committee caches"),
                      ((atts, w.dev, 6), b"unknown fork"), ((atts, w.dev, -1), b"unknown fork")):
        assert call(*args) == _ffi.EINVAL and msg in _ffi.lib.lhb200_last_error(), msg
    assert call(atts, w.dev, rands=np.array([1, 0, 2], dtype=np.uint64)) == _ffi.EINVAL
    assert b"zero random scalar" in _ffi.lib.lhb200_last_error()
    assert call(atts, w.dev, offs=np.array([0, 300, 200, 900], dtype=np.uint64)) == _ffi.EINVAL
    assert b"not monotone" in _ffi.lib.lhb200_last_error()
    total = sum(len(A.index_attestation(a, False, w.host, w.n, FORK_AT_CURRENT, GVR)[1]) for a in atts)
    assert call(atts, w.dev, cap=total - 1) == _ffi.EINVAL and b"indices_cap" in _ffi.lib.lhb200_last_error()
    assert call(atts, w.dev, cap=total) == _ffi.OK
    # the device cache refuses as the host-copy call does
    with pytest.raises(_ffi.Lhb200Error) as exc:
        w.state.device_committee_cache(EPOCH + 2)
    assert exc.value.code == _ffi.EINVAL and b"out of bounds" in _ffi.lib.lhb200_last_error()


def test_no_device_gives_enodev():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    out = C.c_void_p()
    assert _ffi.lib.lhb200_state_committee_cache_create(None, 0, C.byref(out)) == _ffi.ENODEV
    ok, st = C.c_uint8(), np.zeros(1, dtype=np.uint8)
    offs = np.array([0, 229], dtype=np.uint64)
    f = _ffi.Fork()
    assert _ffi.lib.lhb200_attestations_verify(bytes(229), offs.ctypes.data, 1, 4, None, 1, None, C.byref(f), bytes(32),
                                               None, C.byref(ok), st.ctypes.data, None, None, None, 0) == _ffi.ENODEV
    assert _ffi.lib.lhb200_committee_cache_release(None) == _ffi.OK
