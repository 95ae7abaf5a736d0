"""Phase0 (Base) BeaconStates as test and measurement code handles them (no GPU, no pytest): the golden genesis states,
a Base state split into and joined from its field bytes, a chain model of its two pending-attestation lists, and the
from-spec roots of tests/ssz_spec.py memoised so that a replay re-hashes on the CPU only what changed."""
import json
import lzma
import os
import struct

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic
from tests import ssz_spec

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BASE = S.BeaconStateBase
# mainnet BeaconState fixed-part offsets (the same in every fork): slot, block_roots, state_roots, the balances offset,
# the previous_epoch_attestations offset
O_SLOT, O_BLOCK_ROOTS, O_STATE_ROOTS, O_BAL_OFF, O_PP_OFF = 40, 176, 262320, 524556, 2687248


def genesis_state(net):
    """SSZ of the `net` genesis BeaconState: the golden bytes around the validators list, and the validators."""
    meta = json.load(open(os.path.join(GOLDEN, "genesis_states.json")))[net]
    with lzma.open(os.path.join(GOLDEN, f"genesis_state_rest_{net}.bin.xz")) as f:
        rest = f.read()
    with lzma.open(os.path.join(GOLDEN, f"genesis_validators_{net}.bin.xz")) as f:
        vals = f.read()
    o = meta["validators_offset"]
    ssz = rest[:o] + vals + rest[o:]
    assert len(ssz) == meta["ssz_bytes"] and len(vals) == 121 * meta["n_validators"]
    return ssz, meta


def genesis_block(state_root):
    """BeaconBlockBase{slot 0, proposer_index 0, parent_root 0, state_root, empty body}: a genesis block."""
    body = {"randao_reveal": bytes(96), "eth1_data": {"deposit_root": bytes(32), "deposit_count": 0,
                                                      "block_hash": bytes(32)},
            "graffiti": bytes(32), "proposer_slashings": [], "attester_slashings": [], "attestations": [],
            "deposits": [], "voluntary_exits": []}
    return {"slot": 0, "proposer_index": 0, "parent_root": bytes(32), "state_root": state_root, "body": body}


def split_fields(ssz):
    """The SSZ bytes of every field of a Base state."""
    fixed, var, pos = [], [], 0
    for name, ft in BASE[1]:
        if S.is_fixed(ft):
            fixed.append((pos, pos + S.fixed_size(ft)))
            pos += S.fixed_size(ft)
        else:
            var.append(len(fixed))
            fixed.append(struct.unpack_from("<I", ssz, pos)[0])
            pos += 4
    offs = [fixed[i] for i in var] + [len(ssz)]
    out = []
    for i, f in enumerate(fixed):
        if i in var:
            k = var.index(i)
            out.append(bytes(ssz[offs[k]:offs[k + 1]]))
        else:
            out.append(bytes(ssz[f[0]:f[1]]))
    return out


def split_records(b):
    """The records of a List[PendingAttestation, 4096]'s SSZ."""
    if not b:
        return []
    n = struct.unpack_from("<I", b, 0)[0] // 4
    offs = [struct.unpack_from("<I", b, 4 * i)[0] for i in range(n)] + [len(b)]
    return [bytes(b[offs[i]:offs[i + 1]]) for i in range(n)]


def join_fields(fields):
    """SSZ of a Base state from the bytes of its 21 fields."""
    fixed, tail = [], []
    at = sum(S.fixed_size(ft) if S.is_fixed(ft) else 4 for _, ft in BASE[1])
    for (name, ft), b in zip(BASE[1], fields):
        if S.is_fixed(ft):
            fixed.append(b)
        else:
            fixed.append(struct.pack("<I", at))
            tail.append(b)
            at += len(b)
    return b"".join(fixed + tail)


def with_pending(ssz, prev, cur):
    """The state `ssz` with its pending-attestation lists replaced."""
    f = split_fields(ssz)
    f[15], f[16] = prev, cur
    return join_fields(f)


class SpecRoots:
    """From-spec field roots of Base states, memoised by each field's bytes (and each pending record's)."""

    def __init__(self):
        self.memo = {}

    def _cached(self, key, fn):
        if key not in self.memo:
            self.memo[key] = fn()
        return self.memo[key]

    def record_root(self, r):
        return self._cached(("rec", r), lambda: ssz_spec.hash_tree_root(
            S.PendingAttestation, ssz_spec.deserialize(S.PendingAttestation, r)))

    def pending_root(self, b):
        recs = split_records(b)
        return ssz_spec.mix_in_length(ssz_spec.merkleize([self.record_root(r) for r in recs], 4096), len(recs))

    def fields(self, ssz):
        out = []
        for (name, ft), b in zip(BASE[1], split_fields(ssz)):
            if name.endswith("_epoch_attestations"):
                out.append(self._cached((name, b), lambda b=b: self.pending_root(b)))
            else:
                out.append(self._cached((name, b), lambda ft=ft, b=b: ssz_spec.hash_tree_root(
                    ft, ssz_spec.deserialize(ft, b))))
        return out

    def root(self, ssz):
        f = self.fields(ssz)
        return ssz_spec.merkleize(f), f


class Chain:
    """A Base state as the bytes of its fields, and the records of its two pending lists."""

    def __init__(self, ssz):
        self.f = split_fields(ssz)
        self.prev, self.cur = split_records(self.f[15]), split_records(self.f[16])

    def full(self):
        lst = synthetic.pending_attestations_list_ssz
        return join_fields(self.f[:15] + [lst(self.prev), lst(self.cur)] + self.f[17:])

    def balances_offset(self):
        return struct.unpack_from("<I", self.full(), O_BAL_OFF)[0]

    def patch(self, edits):
        full = bytearray(self.full())
        for off, b in edits:
            full[off:off + len(b)] = b
        self.f = split_fields(bytes(full))
