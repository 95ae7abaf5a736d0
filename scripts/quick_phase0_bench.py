"""Phase0 (Base) workloads on one GPU; prints one JSON line with the card name and power limit read in the same run.

  genesis    cold root of the mainnet genesis state (5.4 MB SSZ, 21 063 validators) end to end: stage, root, release;
             checked against its golden root
  blocks     backfill-shaped batches of 64 and 1024 phase0 blocks with 128 attestations each, in blocks/s, next to
             Altair blocks of the same shape (64 distinct blocks, repeated to fill the larger batch)
  replay     a phase0 epoch replay at 250 000 validators: per slot a patch batch (slot, block and state roots, 64
             balances), set_pending_attestations of the current list with the block's 128 attestations appended, and a
             warm root; the epoch rotation (two more calls) at the boundary.  Median and p99 per slot, host clock (the
             root synchronises); roots checked against tests/ssz_spec.py at sampled slots."""
import json
import os
import struct
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import synthetic, tree_hash as T
from tests.phase0_state import O_BLOCK_ROOTS, O_SLOT, O_STATE_ROOTS, Chain, SpecRoots, genesis_state

N_VALIDATORS, N_SLOTS, START = 250_000, 40, 32 * 1000 + 24


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(xs):
    xs = np.array(xs)
    return {"median_ms": round(float(np.median(xs)), 3), "p99_ms": round(float(np.percentile(xs, 99)), 3)}


def genesis():
    ssz, meta = genesis_state("mainnet")
    want = bytes.fromhex(meta["state_root"])
    ms = []
    for _ in range(12):
        t0 = time.perf_counter()
        r = T.beacon_state_root(ssz, "base")
        ms.append(1e3 * (time.perf_counter() - t0))
        assert r == want
    return stats(ms[2:])


def blocks():
    out = {}
    for fork in ("base", "altair"):
        blks = [synthetic.beacon_block_deneb(seed=300 + i, fork=fork, n_attestations=128)[1] for i in range(64)]
        for n in (64, 1024):
            batch = (blks * (n // 64))[:n]
            T.beacon_block_roots(batch, fork)
            ms = []
            for _ in range(8):
                t0 = time.perf_counter()
                T.beacon_block_roots(batch, fork)
                ms.append(1e3 * (time.perf_counter() - t0))
            out[f"{fork}_{n}_blocks_per_s"] = round(n / (float(np.median(ms)) / 1e3))
    return out


def replay():
    lst = synthetic.pending_attestations_list_ssz
    ssz = bytearray(synthetic.beacon_state_deneb_ssz(N_VALIDATORS, seed=5, fork="base", n_hist_roots=2, n_votes=3,
                                                     n_pending_attestations=(4096, 24 * 128),
                                                     pending_bit_lengths=(120, 122, 125)))
    struct.pack_into("<Q", ssz, O_SLOT, START - 1)
    chain, spec = Chain(bytes(ssz)), SpecRoots()
    st = T.ResidentState(bytes(ssz), "base")
    st.enable_incremental()
    st.root()
    rng = np.random.default_rng(9)
    ms, checked = [], 0
    try:
        for k in range(N_SLOTS):
            slot = START + k
            o_bal = chain.balances_offset()
            edits = [(O_SLOT, struct.pack("<Q", slot)), (O_BLOCK_ROOTS + 32 * (slot % 8192), rng.bytes(32)),
                     (O_STATE_ROOTS + 32 * (slot % 8192), rng.bytes(32))]
            edits += [(o_bal + 8 * int(i), rng.bytes(8)) for i in rng.choice(N_VALIDATORS, size=64, replace=False)]
            new = [synthetic.pending_attestation_ssz(rng, 122, slot) for _ in range(128)]
            rotate = slot % 32 == 0
            t0 = time.perf_counter()
            if rotate:
                st.set_pending_attestations(15, lst(chain.cur))
                st.set_pending_attestations(16, b"")
            st.patch_batch(edits)
            st.set_pending_attestations(16, lst(([] if rotate else chain.cur) + new))
            root = st.root()
            ms.append(1e3 * (time.perf_counter() - t0))
            if rotate:
                chain.prev, chain.cur = chain.cur, []
            chain.patch(edits)
            chain.cur = chain.cur + new
            if k % 8 == 0 or rotate or k == N_SLOTS - 1:
                assert root == spec.root(chain.full())[0], slot
                checked += 1
    finally:
        st.release()
    return dict(stats(ms), slots=N_SLOTS, slots_checked=checked)


def main():
    lighthouse_b200.init(0)
    print(json.dumps({"card": card(), "genesis_mainnet_cold_root": genesis(), **blocks(),
                      "epoch_replay_250k": replay()}))


if __name__ == "__main__":
    main()
