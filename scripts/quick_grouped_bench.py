"""Grouped against ungrouped BLS batch verification on batches whose sets share messages.

The driver prints the card (name, SM count, power limit), then runs one worker subprocess per round and mode,
alternating the default (grouping on) and LHB_GROUP_MESSAGES=0 on identical seeded inputs, and prints one JSON line per
workload, mode and round.  Each worker times, after a warm-up:
  * the staged resident path: enqueue -> result on one stream, CUDA events, per step;
  * the plugin call lhb200_verify_signature_sets with pinned host buffers, wall clock per call;
  * for the 64-set gossip batches also 16 threads looping on their own batches through the plugin call (batches/s).
Every line carries a digest of the outputs (verdict, statuses, GT value of the valid batch and of a batch whose sets
all contribute), so the two modes can be checked for identical results.

    python scripts/quick_grouped_bench.py [--steps 20] [--warmup 3] [--rounds 2] [--only name,...]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

V = 16384
# name -> (sets, keys per set, distinct messages); "one_repeat" is the policy's worst case: one message occurs twice
WORKLOADS = {
    "gossip_64x1_1msg": (64, 1, 1),
    "gossip_64x1_4msgs": (64, 1, 4),
    "gossip_64x1_16msgs": (64, 1, 16),
    "sync_512x1_1msg": (512, 1, 1),
    "epoch_100000x128_2048msgs": (100_000, 128, 2048),
    "one_repeat_100000x128": (100_000, 128, 99_999),
}


def stats(ms):
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "steps": len(ms)}


def make_inputs(bls, S, pk_table, n, kps, k, seed):
    import numpy as np
    rng = np.random.default_rng(seed)
    pool = [rng.integers(0, 256, size=32, dtype=np.uint8).tobytes() for _ in range(k)]
    assign = np.arange(n) % k if k < n else np.arange(n)
    if k == n - 1:                                            # one repeat: the last set takes the first set's message
        assign = np.concatenate([np.arange(n - 1), [0]])
    else:
        rng.shuffle(assign)
    work = S.sets_workload(np.full(n, kps), V, seed=seed)
    work["msgs"] = b"".join(pool[g] for g in assign)
    ab = S.materialize_sets(work, pk_table, bls.sign)
    contrib = b"".join(pool[(g + 1) % k] for g in assign) if k > 1 else bytes([pool[0][0] ^ 1]) + pool[0][1:]
    if k == 1:
        contrib = contrib * n
    rands = rng.integers(1, 2 ** 63, size=n, dtype=np.uint64) * 2 + 1
    return ab, contrib, rands


def worker(args):
    import numpy as np
    import torch
    import lighthouse_b200
    from lighthouse_b200 import bls, _ffi
    from lighthouse_b200 import synthetic as S
    lighthouse_b200.init(0)
    lib = _ffi.lib
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    pk_table = S.interop_pubkey_table(V)
    pin = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).pin_memory()
    vp = lambda t: C.c_void_p(t.data_ptr())
    okb = C.create_string_buffer(1)
    mode = "off" if os.environ.get("LHB_GROUP_MESSAGES") == "0" else "grouped"
    for name, (n, kps, k) in WORKLOADS.items():
        if args.only and name not in args.only:
            continue
        ab, contrib, rands = make_inputs(bls, S, pk_table, n, kps, k, seed=0x6B00 + n + k)
        b = bls.Batch(n, n * kps)
        digest = hashlib.sha256()
        b.upload(ab.sigs, contrib, ab.pks, ab.offsets, rands)
        b.enqueue(sp)
        ok_c, st_c = b.result(sp, want_status=True)
        digest.update(bytes([ok_c]) + st_c.tobytes() + b.gt_bytes())
        b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, rands)
        plan = b.plan()
        ms = []
        for step in range(args.warmup + args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            b.enqueue(sp)
            ok, st = b.result(sp, want_status=True)
            e1.record(stream)
            e1.synchronize()
            assert ok
            if step >= args.warmup:
                ms.append(e0.elapsed_time(e1))
        digest.update(bytes([ok]) + st.tobytes() + b.gt_bytes())
        b.destroy()
        h = [pin(ab.sigs), pin(ab.msgs), pin(ab.pks), torch.from_numpy(ab.offsets.astype(np.uint32)).pin_memory(),
             torch.from_numpy(rands.copy()).pin_memory()]
        call = lambda: lib.lhb200_verify_signature_sets(*[vp(t) for t in h], n, okb, None)
        wall = []
        for step in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            _ffi.check(call(), "lhb200_verify_signature_sets")
            if step >= args.warmup:
                wall.append((time.perf_counter() - t0) * 1e3)
            assert okb.raw[0] == 1
        row = {"workload": name, "mode": mode, "sets": n, "keys_per_set": kps, "messages": k, "groups": plan["groups"],
               "hash": plan["hash"], "miller": plan["miller"], "resident": stats(ms), "plugin_pinned": stats(wall),
               "outputs_sha256": digest.hexdigest()}
        if n == 64:
            T, seconds = 16, 1.5
            data = [make_inputs(bls, S, pk_table, n, kps, k, seed=0x6C00 + t)[0] for t in range(T)]
            counts = [0] * T
            stop = [0.0]

            def loop(t):
                a = data[t]
                bls.verify_signature_sets_raw(a.sigs, a.msgs, a.pks, a.offsets)
                while time.perf_counter() < stop[0]:
                    assert bls.verify_signature_sets_raw(a.sigs, a.msgs, a.pks, a.offsets)
                    counts[t] += 1
            stop[0] = time.perf_counter() + seconds
            t0 = time.perf_counter()
            th = [threading.Thread(target=loop, args=(t,)) for t in range(T)]
            [x.start() for x in th]
            [x.join() for x in th]
            row["threads16_batches_per_s"] = sum(counts) / (time.perf_counter() - t0)
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--only", type=lambda s: set(s.split(",")), default=None)
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    import torch
    print(json.dumps({"gpu": q, "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
    base = [sys.executable, os.path.abspath(__file__), "--worker", "--steps", str(args.steps), "--warmup", str(args.warmup)]
    if args.only:
        base += ["--only", ",".join(sorted(args.only))]
    for r in range(args.rounds):
        for env in ({}, {"LHB_GROUP_MESSAGES": "0"}):
            out = subprocess.run(base, env=dict(os.environ, **env), capture_output=True, text=True)
            if out.returncode:
                sys.exit(out.stderr[-3000:])
            for line in out.stdout.splitlines():
                if line.startswith("{"):
                    row = json.loads(line)
                    row["round"] = r
                    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
