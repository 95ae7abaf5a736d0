"""Committee cache, proposer and sync-committee calls on resident BeaconStates; prints one JSON line with the card name
and power limit read in the same run.

For Deneb and Electra states of 500 000 and 1 000 000 validators (all active, synthetic bytes of
lighthouse_b200.synthetic, slot in epoch 300) it first checks the device's shuffling, positions, seed, proposers and
sync indices against the restatement of tests/committee_spec.py, then times:
  cache_ms         ResidentState.committee_cache(epoch) end to end (host clock; the call ends in a synchronise)
  cache_kernels_ms device time of the call's kernels, summed from a torch.profiler run of its own (CUDA activities)
  proposers_ms     beacon_proposer_indices(), end to end
  sync_ms          next_sync_committee_indices(), end to end
  cpu_restatement_ms  the same committee work on the CPU: numpy active scan + the C oracle's shuffle_list (a
                   restatement of the spec, not Lighthouse)
  shuffle_list_ms  lhb200_shuffle_list over the host-computed active set and seed, fed from host buffers
Medians over REPS calls after WARMUP calls."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import _ffi, tree_hash as T
from lighthouse_b200.synthetic import beacon_state_deneb_ssz
from tests import committee_spec as CS
from tests import oracle_lib as O

EPOCH, WARMUP, REPS = 300, 3, 20
KERNELS = ("k_committee_seeds", "k_active_count", "k_active_write", "k_shuffle_hashes", "k_shuffle_permute",
           "k_shuffling_positions")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def median_ms(fn):
    for _ in range(WARMUP):
        fn()
    ms = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return round(float(np.median(ms)), 3)


def kernel_ms(fn, calls=10):
    """Device time per call of the committee kernels, from a profiler trace of `calls` calls."""
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


def run(fork, n):
    ssz = bytearray(beacon_state_deneb_ssz(n, seed=n + 1, fork=fork, n_votes=0, n_hist_roots=0, n_summaries=0))
    CS.set_slot(ssz, EPOCH * 32 + 5)
    ssz = bytes(ssz)
    s = CS.State(ssz)
    h = T.ResidentState(ssz, fork)
    want = CS.committee_cache(s, EPOCH)
    got = h.committee_cache(EPOCH)
    assert np.array_equal(got.shuffling(), want["shuffling"]) and np.array_equal(got._positions, want["positions"])
    assert got.seed == want["seed"] and got.committees_per_slot() == want["committees_per_slot"]
    assert h.beacon_proposer_indices() == CS.beacon_proposer_indices(s)
    assert h.next_sync_committee_indices() == CS.next_sync_committee_indices(s)
    active = CS.active_indices(s, EPOCH)
    seed = want["seed"]
    out = np.empty_like(active)

    def cpu():
        a = CS.active_indices(s, EPOCH)
        O.shuffle_list(a, 90, seed, False)

    def host_shuffle():
        rc = _ffi.lib.lhb200_shuffle_list(C.c_void_p(active.ctypes.data), len(active), 90, seed, 0,
                                          C.c_void_p(out.ctypes.data))
        assert rc == 0
    r = {"fork": fork, "validators": n, "committees_per_slot": want["committees_per_slot"],
         "cache_ms": median_ms(lambda: h.committee_cache(EPOCH)),
         "proposers_ms": median_ms(h.beacon_proposer_indices),
         "sync_ms": median_ms(h.next_sync_committee_indices),
         "shuffle_list_ms": median_ms(host_shuffle),
         "cpu_restatement_ms": median_ms(cpu)}
    host_shuffle()
    assert np.array_equal(out, want["shuffling"])
    r["cache_kernels_ms"] = kernel_ms(lambda: h.committee_cache(EPOCH))
    h.release()
    return r


def main():
    lighthouse_b200.init(0)
    rows = [run(fork, n) for fork in ("deneb", "electra") for n in (500_000, 1_000_000)]
    print(json.dumps({"bench": "committees", "card": card(), "rows": rows}))


if __name__ == "__main__":
    main()
