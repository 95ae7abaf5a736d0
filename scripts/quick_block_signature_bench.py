"""lhb200_block_signatures_verify at 500 000 validators against the route it replaces; prints one JSON line with the
card name and power limit read in the same run.

A Deneb (Electra) state at epoch 300 carries the interop keys in its validator records, a pubkey table holds them, and
device committee caches of epochs 299 and 300 serve the attestations.  Mainnet-like blocks at slots of epoch 300, every
signature valid: 128 aggregate attestations of the previous epoch (Electra: 8, each over 8 committees), one proposer and
one attester slashing, 2 exits, a sync aggregate with about 90 % participation and 2 BLS-to-execution changes.
  deneb1          1 block (SignatureVerifiedBlock::new)
  deneb1_gossip   the same block with LHB200_BLOCK_SKIP_PROPOSAL (the gossip path)
  deneb32         a 32-block segment (signature_verify_chain_segment)
  electra8        8 Electra blocks (+ one consolidation each)
Each row first checks verdict, block statuses and the whole sets table against tests/block_signature_spec.py, then
times:
  call_ms             verify_block_signatures end to end (host clock; the call ends in a synchronise)
  state_front_ms      device time per call of the proposer draw and k_sync_committee_resolve (torch.profiler)
  roots_index_ms      device time per call of k_block_set_roots, the changes' key decoding and the attestation
                      count and write kernels (torch.profiler)
  floor_ms            Batch.upload_indexed + verify fed the restatement's ready sets (the BLS-to-execution changes
                      left out: their keys are not in the table)
  host_route_ms       the restatement's construction (hashlib + numpy, not Lighthouse) plus that upload and verify
Medians over REPS calls after WARMUP calls (host_route_ms: 3)."""
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import bls, block_signatures as BS, tree_hash as T
from lighthouse_b200 import synthetic as SY
from tests import block_signature_spec as B
from tests import committee_spec as CS

N, EPOCH, WARMUP, REPS = 500_000, 300, 3, 10
STATE_FORK = (bytes.fromhex("04000000"), bytes.fromhex("05000000"), 0)
VERSIONS = (bytes.fromhex("00000000"), bytes.fromhex("03000000"))
FRONT = ("k_committee_seeds", "k_active_count", "k_active_write", "k_sample_validators", "k_sync_committee_resolve")
ROOTS = ("k_block_set_roots", "k_g1_decompress_validate", "k_table_import", "k_attestation_index_count",
         "k_attestation_index_write")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def median_ms(fn, reps=REPS):
    for _ in range(WARMUP):
        fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return round(float(np.median(ms)), 3)


def kernel_ms(fn, calls=5):
    """device time per call of the FRONT and ROOTS kernels"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
    tot = {"front": 0.0, "roots": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", 0)   # microseconds
        if any(k in e.key for k in FRONT):
            tot["front"] += t
        elif any(k in e.key for k in ROOTS):
            tot["roots"] += t
    return round(tot["front"] / 1e3 / calls, 4), round(tot["roots"] / 1e3 / calls, 4)


class World:
    def __init__(self, fork, sks, pk48, table):
        ssz = SY.block_signature_state(N, fork, EPOCH * 32 + 20, STATE_FORK, pk48)
        self.fork, self.sks, self.table = fork, sks, table
        self.state = T.ResidentState(ssz, fork)
        self.view = B.StateView(ssz, fork)
        s = CS.State(ssz)
        self.host = [CS.committee_cache(s, e) for e in (EPOCH - 1, EPOCH)]
        self.dev = [self.state.device_committee_cache(e) for e in (EPOCH - 1, EPOCH)]

    def blocks(self, n_blocks):
        from lighthouse_b200.committees import CommitteeCache
        c = self.host[0]
        hc = CommitteeCache(c["epoch"], c["shuffling"], c["positions"], c["committees_per_slot"], c["seed"])
        electra = self.fork == "electra"
        out, roots = [], []
        for k in range(n_blocks):
            slot = EPOCH * 32 + k
            if electra:
                atts = SY.signed_attestations(hc, "electra", 8, self.sks, STATE_FORK, self.view.gvr, seed=k,
                                              committees_per_attestation=8, fill=0.9)
            else:
                atts = SY.signed_attestations(hc, "aggregate", 128, self.sks, STATE_FORK, self.view.gvr, seed=k,
                                              fill=0.9)
            b, r = SY.signed_beacon_block(self.fork, slot, self.view.proposers[slot % 32], self.sks, STATE_FORK,
                                          self.view.gvr, VERSIONS, lambda m: T.beacon_block_roots([m], self.fork)[0],
                                          seed=k, attestations=atts, sync_committee=self.view.sync, n_validators=N)
            out.append(b)
            roots.append(r)
        return out, roots


def restate(w, blks, roots, skip):
    """the host route's preparation: the sets with keys in the table, as Batch.upload_indexed inputs"""
    sets = B.segment(blks, w.fork, w.view, w.host, N, VERSIONS, roots, skip)[0]
    sets = [x for x in sets if x["kind"] != B.BLS_CHANGE]
    idx = np.array([k for x in sets for k in x["keys"]], dtype=np.uint32)
    offs = np.cumsum([0] + [len(x["keys"]) for x in sets]).astype(np.uint32)
    return sets, b"".join(x["signature"] for x in sets), b"".join(x["root"] for x in sets), idx, offs


def row(name, w, blks, roots, skip=False):
    want, want_st, _ = B.segment(blks, w.fork, w.view, w.host, N, VERSIONS, roots, skip)
    ok, st, sets = BS.verify_block_signatures(blks, w.fork, w.state, w.dev, w.table, VERSIONS, roots, None, skip)
    assert ok and st.tolist() == want_st == [0] * len(blks)
    assert [(s[0], s[1], s[2], s[3], s[4]) for s in sets] == \
        [(x["block"], x["item"], x["kind"], x["status"], x["root"]) for x in want]
    sets_, sigs, msgs, idx, offs = restate(w, blks, roots, skip)
    b = bls.Batch(len(sets_), 1)

    def floor():
        b.upload_indexed(w.table, sigs, msgs, idx, offs)
        b.enqueue()
        assert b.result()

    def host_route():
        _, s_, m_, i_, o_ = restate(w, blks, roots, skip)
        b.upload_indexed(w.table, s_, m_, i_, o_)
        b.enqueue()
        assert b.result()

    call = lambda: BS.verify_block_signatures(blks, w.fork, w.state, w.dev, w.table, VERSIONS, roots, None, skip)
    front, roots_index = kernel_ms(call)
    r = {"workload": name, "blocks": len(blks), "sets": len(sets), "table_keys": int(offs[-1]),
         "call_ms": median_ms(call), "state_front_ms": front, "roots_index_ms": roots_index,
         "floor_ms": median_ms(floor), "host_route_ms": median_ms(host_route, reps=3)}
    b.destroy()
    return r


def main():
    lighthouse_b200.init(0)
    sks = SY.interop_secret_keys(N)
    pk48, pk96 = bls.sk_to_pk(b"".join(s.to_bytes(32, "big") for s in sks))
    table = bls.PubkeyTable(N)
    table.append(pk96)
    rows = []
    w = World("deneb", sks, pk48, table)
    blks, roots = w.blocks(32)
    rows.append(row("deneb1", w, blks[:1], roots[:1]))
    rows.append(row("deneb1_gossip", w, blks[:1], roots[:1], skip=True))
    rows.append(row("deneb32", w, blks, roots))
    w = World("electra", sks, pk48, table)
    blks, roots = w.blocks(8)
    rows.append(row("electra8", w, blks, roots))
    print(json.dumps({"bench": "block_signatures", "card": card(), "validators": N, "rows": rows}))


if __name__ == "__main__":
    main()
