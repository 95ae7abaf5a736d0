"""The SSZ layouts of every fork the tree-hash path reads (BeaconState and BeaconBlock, full and blinded, Altair ..
Electra), through malformed input and in-place patches.

Malformed input: starting from valid synthetic SSZ, every variable-size part of the object (container fields and the
items of lists of variable-size items, at any depth) gets an offset that is not the fixed size, one below its
predecessor and one past the end; every list of fixed-size items gets a span that is not a whole number of items; and
every list, bit list and byte list whose limit is small enough to build gets one item (bit, byte) over its limit.  The
header's extra_data of 33 bytes is one of those.  Each case must be refused with EINVAL, and the untouched bytes must
give the from-spec root of tests/ssz_spec.py.

Patches: bytes of the fields a staged state keeps as literal chunks (the payload header's logs_bloom and extra_data,
eth1_data, a checkpoint, latest_block_header) are patched on a resident state of each fork; the root must equal the
from-spec root of the patched bytes, cold and with the incremental path enabled."""
import ctypes as C
import struct

import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic
from tests import ssz_spec

pytestmark = pytest.mark.gpu

FORKS = ["altair", "bellatrix", "capella", "deneb", "electra"]
MAX_CASE_BYTES = 8 << 20   # over-limit lists larger than this are not built (validators, historical roots, ...)


def _u32(b, at):
    return int.from_bytes(b[at:at + 4], "little")


def _var_parts(t, b):
    """[key, type, start, end, position of the offset] of each variable-size part of SSZ bytes `b` of type `t`: the
    variable fields of a container, the items of a list of variable-size items."""
    if t[0] == "container":
        parts, pos = [], 0
        for name, ft in t[1]:
            if S.is_fixed(ft):
                pos += S.fixed_size(ft)
            else:
                parts.append([name, ft, _u32(b, pos), None, pos])
                pos += 4
    elif t[0] == "list" and not S.is_fixed(t[1]):
        parts = [[i, t[1], _u32(b, 4 * i), None, 4 * i] for i in range(_u32(b, 0) // 4 if b else 0)]
    else:
        return []
    for i, p in enumerate(parts):
        p[3] = parts[i + 1][2] if i + 1 < len(parts) else len(b)
    return parts


def _walk(t, b, path=()):
    """(path, type, bytes) of every variable-size part below `t`; of the items of a list only the first and last."""
    parts = _var_parts(t, b)
    if t[0] == "list":
        parts = [p for p in parts if p[0] in (0, len(parts) - 1)]
    for key, ft, s, e, _ in parts:
        yield path + (key,), ft, b[s:e]
        yield from _walk(ft, b[s:e], path + (key,))


def _replace(t, b, path, raw):
    """SSZ `b` of type `t` with the variable-size part at `path` replaced by `raw`, the enclosing offsets moved to
    match."""
    parts = _var_parts(t, b)
    tails = [(raw if len(path) == 1 else _replace(ft, b[s:e], path[1:], raw)) if key == path[0] else b[s:e]
             for key, ft, s, e, _ in parts]
    head, at = bytearray(b[:parts[0][2]]), parts[0][2]
    for (_, _, _, _, pos), tail in zip(parts, tails):
        head[pos:pos + 4] = struct.pack("<I", at)
        at += len(tail)
    return bytes(head) + b"".join(tails)


def _set_offset(t, b, path, value):
    """SSZ `b` of type `t` with the offset of the variable-size part at `path` set to `value`."""
    base, span = 0, b
    for key in path:
        _, t, s, e, pos = next(p for p in _var_parts(t, span) if p[0] == key)
        at, base, span = base + pos, base + s, span[s:e]
    out = bytearray(b)
    out[at:at + 4] = struct.pack("<I", value)
    return bytes(out)


def _over_limit(ft, span):
    """Bytes of `ft` with one element more than its limit, or None when that is too large to build."""
    k = ft[0]
    if k == "bytelist":
        return bytes(ft[1] + 1) if ft[1] + 1 <= MAX_CASE_BYTES else None
    if k == "bitlist":
        return S.pack_bits([True] * (ft[1] + 1), True) if ft[1] // 8 <= MAX_CASE_BYTES else None
    n = ft[2] + 1
    if S.is_fixed(ft[1]):
        sz = S.fixed_size(ft[1])
        return (span[:sz] if span else bytes(sz)) * n if n * sz <= MAX_CASE_BYTES else None
    parts = _var_parts(ft, span)
    if ft[1][0] == "bytelist":
        item = b""
    elif parts:
        item = span[parts[0][2]:parts[0][3]]
    else:
        return None
    if n * (4 + len(item)) > MAX_CASE_BYTES:
        return None
    return b"".join(struct.pack("<I", 4 * n + i * len(item)) for i in range(n)) + item * n


def malformed(t, ssz):
    """(label, SSZ) of every malformed case derived from the valid `ssz` of type `t`."""
    out = []
    for path, ft, span in [((), t, ssz)] + list(_walk(t, ssz)):
        name = ".".join(map(str, path)) or "<top>"
        parts = _var_parts(ft, span)
        if parts:
            out.append((f"{name}: first offset not the fixed size",
                        _set_offset(t, ssz, path + (parts[0][0],), parts[0][2] + 1)))
            for i, (key, _, _, _, _) in enumerate(parts):
                if ft[0] == "list" and i not in (1, len(parts) - 1):
                    continue
                if i:
                    out.append((f"{name}.{key}: offset below its predecessor",
                                _set_offset(t, ssz, path + (key,), parts[i - 1][2] - 1)))
                out.append((f"{name}.{key}: offset past the end", _set_offset(t, ssz, path + (key,), len(span) + 1)))
        if not path:
            continue
        if ft[0] == "list" and S.is_fixed(ft[1]) and S.fixed_size(ft[1]) > 1:
            out.append((f"{name}: not a whole number of items", _replace(t, ssz, path, span + b"\0")))
        if ft[0] in ("list", "bitlist", "bytelist"):
            raw = _over_limit(ft, span)
            if raw is not None:
                out.append((f"{name}: one over the limit", _replace(t, ssz, path, raw)))
    return out


def _blind(fork, value):
    """The blinded form of a block value: the payload replaced by its header (list fields -> their roots)."""
    import copy
    pt = dict(S.EXECUTION_PAYLOAD_BY_FORK[fork][1])
    v = copy.deepcopy(value)
    p = v["body"]["execution_payload"]
    v["body"]["execution_payload"] = {
        n: p[n] if n in p else ssz_spec.hash_tree_root(pt[n[:-len("_root")]], p[n[:-len("_root")]])
        for n, _ in S.EXECUTION_PAYLOAD_HEADER_BY_FORK[fork][1]}
    return v


def _blocks(fork):
    """(label, type, value, SSZ) of a small block of `fork` with every list non-empty, and its blinded form."""
    if fork == "electra":
        value, _ = synthetic.beacon_block_electra(seed=90, n_attestations=2, committees_per_attestation=2,
                                                  bits_per_committee=30, n_deposit_requests=2, n_withdrawal_requests=2,
                                                  n_transactions=3, n_withdrawals=2, n_blobs=2, slashing_indices=5)
    else:
        value, _ = synthetic.beacon_block_deneb(seed=90, fork=fork, n_attestations=2, n_transactions=3, committee=20,
                                                n_withdrawals=2, n_blobs=2, n_exits=1, n_bls_changes=1)
    out = [("full", S.BEACON_BLOCK_BY_FORK[fork], value)]
    if fork != "altair":
        out.append(("blinded", S.BLINDED_BEACON_BLOCK_BY_FORK[fork], _blind(fork, value)))
    return [(label, t, v, S.serialize(t, v)) for label, t, v in out]


def _expect_einval(fn, cases):
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


@pytest.mark.parametrize("fork", FORKS)
def test_gpu_malformed_blocks_every_fork(gpu, fork):
    from lighthouse_b200 import tree_hash
    for label, t, value, ssz in _blocks(fork):
        blinded = label == "blinded"
        assert tree_hash.beacon_block_roots([ssz], fork, blinded=blinded) == [ssz_spec.hash_tree_root(t, value)]
        cases = malformed(t, ssz)
        assert len(cases) > 40, len(cases)
        _expect_einval(lambda b: tree_hash.beacon_block_roots([b], fork, blinded=blinded), cases)


def _state(fork):
    return synthetic.beacon_state_deneb_ssz(40, seed=91, fork=fork, n_hist_roots=3, n_votes=2, n_summaries=2,
                                            n_pending=(2, 2, 2))


def _spec_state_root(fork, ssz):
    t = S.BEACON_STATE_BY_FORK[fork]
    return ssz_spec.hash_tree_root(t, ssz_spec.deserialize(t, ssz))


@pytest.mark.parametrize("fork", FORKS)
def test_gpu_malformed_states_every_fork(gpu, fork):
    from lighthouse_b200 import tree_hash
    ssz = _state(fork)
    assert tree_hash.beacon_state_root(ssz, fork) == _spec_state_root(fork, ssz)
    cases = malformed(S.BEACON_STATE_BY_FORK[fork], ssz)
    labels = " ".join(label for label, _ in cases)
    assert "eth1_data_votes: one over the limit" in labels
    if fork != "altair":
        assert "latest_execution_payload_header.extra_data: one over the limit" in labels
    _expect_einval(lambda b: tree_hash.beacon_state_root(b, fork), cases)


# mainnet BeaconState fixed-part offsets of the fields patched below (the same in every fork)
O_LBH, O_ETH1_DATA, O_PJC, O_FC = 64, 524468, 2687257, 2687337
HDR_FIXED = {"bellatrix": 536, "capella": 568, "deneb": 584, "electra": 648}


@pytest.mark.parametrize("fork", FORKS)
def test_gpu_state_patch_of_literal_fields_every_fork(gpu, fork):
    from lighthouse_b200._ffi import lib, check, buf
    from lighthouse_b200.tree_hash import FORKS as FORK_IDS
    ssz = bytearray(_state(fork))
    h = C.c_void_p()
    p, keep = buf(bytes(ssz))
    check(lib.lhb200_state_stage(p, len(ssz), FORK_IDS[fork], C.byref(h)), "lhb200_state_stage")

    def root():
        out = C.create_string_buffer(32)
        check(lib.lhb200_state_root(h, out, None), "lhb200_state_root")
        return out.raw

    def patch(off, data):
        ssz[off:off + len(data)] = data
        q, k = buf(data)
        check(lib.lhb200_state_patch(h, off, q, len(data)), "lhb200_state_patch")

    edits = [(O_LBH + 3, b"\x5a"), (O_LBH + 60, b"\xa5\x01"), (O_ETH1_DATA + 5, b"\x77"), (O_ETH1_DATA + 33, b"\x11"),
             (O_PJC + 1, b"\x42"), (O_FC + 20, b"\x24")]
    if fork != "altair":
        o_leph = struct.unpack_from("<I", ssz, 2736629)[0]
        edits += [(o_leph + 116 + 7, b"\xee"), (o_leph + 116 + 255, b"\x3c"), (o_leph + HDR_FIXED[fork] + 2, b"\x99")]
    try:
        assert root() == _spec_state_root(fork, bytes(ssz))
        for off, data in edits[::2]:
            patch(off, data)
        assert root() == _spec_state_root(fork, bytes(ssz))
        check(lib.lhb200_state_enable_incremental(h), "lhb200_state_enable_incremental")
        assert root() == _spec_state_root(fork, bytes(ssz))
        for off, data in edits[1::2]:
            patch(off, data)
        assert root() == _spec_state_root(fork, bytes(ssz))
    finally:
        lib.lhb200_state_release(h)
