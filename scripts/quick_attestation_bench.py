"""lhb200_attestations_verify at 500 000 validators against the route it replaces; prints one JSON line with the card
name and power limit read in the same run.

Workloads over a Deneb (Electra) state at epoch 300 with every validator active, interop keys in a resident pubkey table
and device committee caches of epochs 299 and 300:
  gossip64        64 unaggregated single-bit attestations over 2 committees of one slot (one gossip batch)
  segment4096     4 096 aggregate attestations, every committee of the two epochs once (config 3's 32-block segment)
  electra64x64    Electra: 64 attestations, each over all 64 committees of one slot of the two epochs (the same
                  validators as segment4096)
Each row first checks verdict, statuses, signing roots and indices against tests/attestation_spec.py, then times:
  call_ms           verify_attestations end to end (host clock; the call ends in a synchronise)
  index_kernels_ms  device time of k_attestation_index_count + k_attestation_index_write per call, summed from a
                    torch.profiler trace of its own (CUDA activities)
  host_route_ms     today's route: indices and signing roots from the restatement, then Batch.upload_indexed + verify
  upload_verify_ms  the upload_indexed + verify part of host_route_ms alone
  cpu_restatement_ms  the restatement's indexing and roots alone (hashlib + numpy, not Lighthouse)
Medians over REPS calls after WARMUP calls."""
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import attestations as AT, bls, tree_hash as T
from lighthouse_b200.synthetic import (MAINNET_GVR, beacon_state_deneb_ssz, interop_pubkey_table, interop_secret_keys,
                                       signed_attestations)
from tests import attestation_spec as A
from tests import committee_spec as CS

N, EPOCH, WARMUP, REPS = 500_000, 300, 3, 15
FORK_INFO = (bytes.fromhex("04000000"), bytes.fromhex("05000000"), 0)
KERNELS = ("k_attestation_index_count", "k_attestation_index_write")


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


def kernel_ms(fn, calls=10):
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
    total = 0.0
    for e in prof.key_averages():
        if any(k in e.key for k in KERNELS):
            total += getattr(e, "device_time_total", None) or e.cuda_time_total   # microseconds
    return round(total / 1e3 / calls, 4)


def restate(atts, electra, host):
    """The host route's preparation: statuses, signing roots, key-index CSR of the sets."""
    out = [A.index_attestation(a, electra, host, N, FORK_INFO, MAINNET_GVR) for a in atts]
    idx = np.concatenate([o[1] for o in out]).astype(np.uint32)
    offs = np.zeros(len(out) + 1, dtype=np.uint32)
    np.cumsum([len(o[1]) for o in out], out=offs[1:])
    return out, b"".join(a[132:228] for a in atts), b"".join(o[2] for o in out), idx, offs


def row(name, fork, atts, electra, dev, host, table):
    out, sigs, msgs, idx, offs = restate(atts, electra, host)
    ok, st, roots, ind = AT.verify_attestations(atts, fork, dev, table, FORK_INFO, MAINNET_GVR, want_indices=True)
    assert ok and not st.any()
    assert roots == [o[2] for o in out] and all(a.tolist() == o[1].tolist() for a, o in zip(ind, out))
    b = bls.Batch(len(atts), 1)

    def upload_verify():
        b.upload_indexed(table, sigs, msgs, idx, offs)
        b.enqueue()
        assert b.result()

    def host_route():
        _, s_, m_, i_, o_ = restate(atts, electra, host)
        b.upload_indexed(table, s_, m_, i_, o_)
        b.enqueue()
        assert b.result()

    call = lambda: AT.verify_attestations(atts, fork, dev, table, FORK_INFO, MAINNET_GVR)
    r = {"workload": name, "attestations": len(atts), "keys": int(offs[-1]), "call_ms": median_ms(call),
         "index_kernels_ms": kernel_ms(call), "upload_verify_ms": median_ms(upload_verify),
         "host_route_ms": median_ms(host_route, reps=3),
         "cpu_restatement_ms": median_ms(lambda: restate(atts, electra, host), reps=3)}
    b.destroy()
    return r


def main():
    lighthouse_b200.init(0)
    sks = interop_secret_keys(N)
    table = bls.PubkeyTable(N)
    table.append(interop_pubkey_table(N).tobytes())
    rows = []
    for fork in ("deneb", "electra"):
        ssz = bytearray(beacon_state_deneb_ssz(N, seed=3, fork=fork, n_votes=0, n_hist_roots=0, n_summaries=0))
        CS.set_slot(ssz, EPOCH * 32 + 5)
        state = T.ResidentState(bytes(ssz), fork)
        epochs = (EPOCH - 1, EPOCH)
        dev = [state.device_committee_cache(e) for e in epochs]
        hostc = [d.to_host() for d in dev]
        electra = fork == "electra"
        if electra:
            atts = [a for k, c in enumerate(hostc)
                    for a in signed_attestations(c, "electra", 32, sks, FORK_INFO, seed=k, committees_per_attestation=64)]
            rows.append(row("electra64x64", fork, atts, True, dev, hostc, table))
        else:
            atts = signed_attestations(hostc[1], "unaggregated", 64, sks, FORK_INFO, slot=EPOCH * 32 + 3, n_committees=2)
            rows.append(row("gossip64", fork, atts, False, dev, hostc, table))
            cps = hostc[0].committees_per_slot()
            atts = [a for k, c in enumerate(hostc) for a in signed_attestations(c, "aggregate", 32 * cps, sks, FORK_INFO, seed=k)]
            rows.append(row("segment4096", fork, atts, False, dev, hostc, table))
        for d in dev:
            d.release()
        state.release()
    table.destroy()
    print(json.dumps({"bench": "attestations", "card": card(), "validators": N, "rows": rows}))


if __name__ == "__main__":
    main()
