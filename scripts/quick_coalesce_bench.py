"""Concurrent gossip callers through the plugin call: T threads, each looping its own 64-set batch through
lhb200_verify_signature_sets (host buffers, library-drawn scalars), T in {1, 8, 16, 32, 64}, for 1-key and 128-key
sets.  Prints one JSON line per (keys, T): batches/s, median and p99 call latency, and the card it ran on.
Concurrent calls are coalesced into segmented passes (DESIGN.md §2.7); T = 1 is the lone-call path.

usage: python scripts/quick_coalesce_bench.py [--root TREE] [--seconds S]
    --root: the tree whose lighthouse_b200 is imported (to compare two builds alternately in one session)"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--seconds", type=float, default=2.0)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import lighthouse_b200  # noqa: E402
from lighthouse_b200 import bls  # noqa: E402
from lighthouse_b200.synthetic import attestation_batch, interop_pubkey_table  # noqa: E402

lighthouse_b200.init(0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
N_SETS, N_VAL, THREADS = 64, 2048, (1, 8, 16, 32, 64)
table = interop_pubkey_table(N_VAL)
for keys in (1, 128):
    batches = [attestation_batch(N_SETS, keys_per_set=keys, n_validators=N_VAL, seed=900 + t, pk_table=table)
               for t in range(max(THREADS))]

    def call(t):
        ab = batches[t]
        return bls.verify_signature_sets_raw(ab.sigs, ab.msgs, ab.pks, ab.offsets)

    for T in THREADS:
        warm = [threading.Thread(target=call, args=(t,)) for t in range(T)]   # pooled handles for T callers
        [w.start() for w in warm]
        [w.join() for w in warm]
        lat = [[] for _ in range(T)]
        stop = time.perf_counter() + args.seconds

        def work(t):
            while time.perf_counter() < stop:
                t0 = time.perf_counter()
                assert call(t)
                lat[t].append(time.perf_counter() - t0)

        t0 = time.perf_counter()
        th = [threading.Thread(target=work, args=(t,)) for t in range(T)]
        [x.start() for x in th]
        [x.join() for x in th]
        dt = time.perf_counter() - t0
        all_lat = np.concatenate([np.asarray(x) for x in lat]) * 1e3
        print(json.dumps({"root": os.path.abspath(args.root), "card": card, "keys_per_set": keys, "threads": T,
                          "batches_per_s": len(all_lat) / dt, "sets_per_s": len(all_lat) * N_SETS / dt,
                          "median_ms": float(np.median(all_lat)), "p99_ms": float(np.percentile(all_lat, 99))}),
              flush=True)
