"""A resident 500 000-validator state following a synthetic chain: warm root per slot (arm A) against re-staging the
current bytes and a cold root (arm B), the only way to follow length changes without resizable lists.

64 slots (two epochs) from a seed, per fork (Deneb, Electra):
  every slot     one eth1 vote appended, the payload header replaced (random extra_data length), one slot of
                 committees' participation flags, randao mix, block root, state root, slot and block header patched
  every 4th      16 deposits on the five per-validator lists (plus pending_balance_deposits for Electra)
  epoch boundary every balance, participation rotation, an eth1 reset and a historical_summaries push (first boundary),
                 an Electra pending drain
The arms alternate slot by slot and their roots must agree.  Times are host clocks around the calls, ending in a
device synchronise (lhb200_state_root synchronises); edit = patch_batch + list_edit + set_payload_header only."""
import json
import os
import struct
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import ssz_schema as S, tree_hash as T
from lighthouse_b200.synthetic import beacon_state_deneb_ssz, validators_ssz

N_VALIDATORS, N_SLOTS, SLOTS_PER_EPOCH = 500_000, 64, 32
HEADER_FIXED = {"deneb": 584, "electra": 648}


class Encoding:
    """Fixed part + the bytes of each variable-size field, re-joined with recomputed offsets."""

    def __init__(self, ssz, fork):
        typ = S.BEACON_STATE_BY_FORK[fork]
        self.var, pos = [], 0
        self.item = {}
        for name, ft in typ[1]:
            if S.is_fixed(ft):
                pos += S.fixed_size(ft)
            else:
                self.var.append((name, pos))
                if ft[0] == "list":
                    self.item[name] = S.fixed_size(ft[1])
                pos += 4
        self.fixed = bytearray(ssz[:pos])
        offs = [struct.unpack_from("<I", ssz, p)[0] for _, p in self.var] + [len(ssz)]
        self.parts = {n: bytearray(ssz[offs[i]:offs[i + 1]]) for i, (n, _) in enumerate(self.var)}

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

    def length(self, name):
        return len(self.parts[name]) // self.item[name]

    def edit(self, name, new_len, first, data):
        ib = self.item[name]
        p = self.parts[name]
        p[first * ib:first * ib + len(data)] = data
        del p[new_len * ib:]


def slot_work(rng, enc, fork, slot):
    """(patches, list edits, header) of one slot, applied to `enc` as they are built.  The handle applies the patches
    first, so every patch is built before the first edit and addresses the encoding as the slot found it."""
    patches, edits = [], []

    def fixed(off, data):
        enc.fixed[off:off + len(data)] = data
        patches.append((off, data))

    def var(name, rel, data):
        enc.parts[name][rel:rel + len(data)] = data
        patches.append((enc.offset(name) + rel, data))

    def edit(name, new_len, first, data):
        enc.edit(name, new_len, first, data)
        edits.append((name, new_len, first, data))

    rb = lambda n: rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    fixed(40, struct.pack("<Q", 9000 + slot))                                   # slot
    fixed(64, rb(112))                                                          # latest_block_header
    fixed(524560 + 32 * (slot % 65536), rb(32))                                 # randao mix
    fixed(176 + 32 * (slot % 8192), rb(32))                                     # block root
    fixed(262320 + 32 * (slot % 8192), rb(32))                                  # state root
    nv = enc.length("validators")
    per_slot = nv // SLOTS_PER_EPOCH                                            # one slot of committees
    c0 = (slot % SLOTS_PER_EPOCH) * per_slot
    var("current_epoch_participation", c0, rng.integers(0, 8, size=per_slot, dtype=np.uint8).tobytes())
    boundary = slot % SLOTS_PER_EPOCH == SLOTS_PER_EPOCH - 1
    if boundary:                                                                # every balance (offsets of the
        var("balances", 0, rng.integers(1, 1 << 40, size=nv, dtype="<u8").tobytes())   # encoding before the edits)
    votes = enc.length("eth1_data_votes")
    if boundary and slot < SLOTS_PER_EPOCH:                                     # voting period ends once
        edit("eth1_data_votes", 0, 0, b"")
        edit("historical_summaries", enc.length("historical_summaries") + 1, enc.length("historical_summaries"), rb(64))
    else:
        edit("eth1_data_votes", votes + 1, votes, rb(72))
    if slot % 4 == 0 and not boundary:                                          # 16 deposits
        k = 16
        edit("validators", nv + k, nv, validators_ssz(k, rng))
        edit("balances", nv + k, nv, np.full(k, 32_000_000_000, dtype="<u8").tobytes())
        edit("previous_epoch_participation", nv + k, nv, bytes(k))
        edit("current_epoch_participation", nv + k, nv, bytes(k))
        edit("inactivity_scores", nv + k, nv, bytes(8 * k))
        if fork == "electra":
            m = enc.length("pending_balance_deposits")
            edit("pending_balance_deposits", m + k, m, b"".join(struct.pack("<QQ", nv + i, 32 * 10**9) for i in range(k)))
    if boundary:                                                                # epoch processing
        edit("previous_epoch_participation", nv, 0, bytes(enc.parts["current_epoch_participation"]))
        edit("current_epoch_participation", nv, 0, bytes(nv))
        if fork == "electra":
            m = enc.length("pending_balance_deposits")
            drain = min(m, 64)
            edit("pending_balance_deposits", m - drain, 0, bytes(enc.parts["pending_balance_deposits"][16 * drain:]))
    hdr = bytearray(rb(HEADER_FIXED[fork]))
    hdr[436:440] = struct.pack("<I", HEADER_FIXED[fork])
    hdr = bytes(hdr) + rb(int(rng.integers(0, 33)))
    enc.parts["latest_execution_payload_header"][:] = hdr
    return patches, edits, hdr


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(xs):
    xs = np.array(xs)
    return {"median_ms": round(float(np.median(xs)), 3), "p99_ms": round(float(np.percentile(xs, 99)), 3)}


def run(fork, seed):
    rng = np.random.default_rng(seed)
    ssz = beacon_state_deneb_ssz(N_VALIDATORS, seed=seed, fork=fork, n_votes=3, n_summaries=40)
    enc = Encoding(ssz, fork)
    st = T.ResidentState(ssz, fork)
    st.enable_incremental()
    st.root()
    a_total, a_edit, b_total, warm_hashes = [], [], [], []
    for slot in range(N_SLOTS):
        patches, edits, hdr = slot_work(rng, enc, fork, slot)
        cur = enc.ssz()

        def arm_a():
            t0 = time.perf_counter()
            st.patch_batch(patches)
            st.list_edit(edits)
            st.set_payload_header(hdr)
            t1 = time.perf_counter()
            r = st.root()
            t2 = time.perf_counter()
            a_edit.append((t1 - t0) * 1e3)
            a_total.append((t2 - t0) * 1e3)
            warm_hashes.append(st.last_root_hashes)
            return r

        def arm_b():
            t0 = time.perf_counter()
            r = T.beacon_state_root(cur, fork)
            b_total.append((time.perf_counter() - t0) * 1e3)
            return r

        if slot % 2:
            rb_, ra = arm_b(), arm_a()
        else:
            ra, rb_ = arm_a(), arm_b()
        assert ra == rb_, f"{fork} slot {slot}: warm root differs from the re-staged cold root"
    out = {"warm_per_slot": stats(a_total), "warm_edit_calls": stats(a_edit), "restage_cold_per_slot": stats(b_total),
           "warm_hashes_median": int(np.median(warm_hashes)), "hash_units": int(st.hash_units),
           "validators_at_end": enc.length("validators"), "roots_equal_every_slot": True}
    st.release()
    return out


def main():
    lighthouse_b200.init(0)
    res = {"card": card(), "slots": N_SLOTS, "n_validators": N_VALIDATORS}
    for fork, seed in (("deneb", 1), ("electra", 2)):
        res[fork] = run(fork, seed)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
