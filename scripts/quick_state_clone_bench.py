"""Branching a resident 500 000-validator state: a device clone per slot against the linear warm path and re-staging.

Converted handles of Deneb and Electra follow the 64-slot chain of scripts/quick_warm_chain_bench.py, three ways:
  (a) clone    clone the parent, apply the slot's edits to the clone, warm root, release the parent (how a node
               advances: every state handed out of its cache is a clone)
  (b) linear   the same edits on one handle, warm root (no branching)
  (c) restage  stage the slot's bytes and take a cold root
The arms rotate their order slot by slot and their roots must agree on every slot.  Clone times are host clocks around
lhb200_state_clone, which returns after a device synchronise.  The copy share is the device time of its one
k_copy_ranges launch, read from torch.profiler over extra clones of the final handle; the rest is allocation, the
host-side relocation and the table uploads.  A torch device-to-device copy of the same live byte count, in the same
run, is the bandwidth reference."""
import ctypes as C
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import lighthouse_b200
from lighthouse_b200 import _ffi, tree_hash as T
from lighthouse_b200.synthetic import beacon_state_deneb_ssz
from quick_warm_chain_bench import N_SLOTS, N_VALIDATORS, Encoding, card, slot_work, stats


def live_bytes(st):
    n = C.c_uint64(0)
    _ffi.check(_ffi.lib.lhb200_debug_state_live_bytes(st._h, C.byref(n)), "lhb200_debug_state_live_bytes")
    return n.value


def apply(st, patches, edits, hdr):
    st.patch_batch(patches)
    st.list_edit(edits)
    st.set_payload_header(hdr)


def copy_kernel_ms(st, reps=16):
    """Device time of k_copy_ranges over `reps` clones of `st` (each released at once)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            st.clone().release()
        torch.cuda.synchronize()
    us = [getattr(e, "device_time", None) or e.cuda_time for e in prof.events() if "k_copy_ranges" in e.name]
    return [u / 1e3 for u in us]


def torch_copy_ms(nbytes, reps=20):
    import torch
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    b.copy_(a)
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    del a, b
    torch.cuda.empty_cache()
    return ms


def run(fork, seed):
    rng = np.random.default_rng(seed)
    ssz = beacon_state_deneb_ssz(N_VALIDATORS, seed=seed, fork=fork, n_votes=3, n_summaries=40)
    enc = Encoding(ssz, fork)
    parent, lin = T.ResidentState(ssz, fork), T.ResidentState(ssz, fork)
    for h in (parent, lin):
        h.enable_incremental()
        h.root()
        h.truncate("eth1_data_votes", 3)   # converts: the lists get storage of their own (same encoding)
        h.root()
    clone_ms, a_ms, b_ms, c_ms, live, held = [], [], [], [], [], []
    for slot in range(N_SLOTS):
        patches, edits, hdr = slot_work(rng, enc, fork, slot)
        cur = enc.ssz()
        roots = {}

        def arm_a():
            nonlocal parent
            live.append(live_bytes(parent))
            held.append(parent.device_bytes)
            t0 = time.perf_counter()
            child = parent.clone()
            t1 = time.perf_counter()
            apply(child, patches, edits, hdr)
            roots["a"] = child.root()
            parent.release()
            a_ms.append((time.perf_counter() - t0) * 1e3)
            clone_ms.append((t1 - t0) * 1e3)
            parent = child

        def arm_b():
            t0 = time.perf_counter()
            apply(lin, patches, edits, hdr)
            roots["b"] = lin.root()
            b_ms.append((time.perf_counter() - t0) * 1e3)

        def arm_c():
            t0 = time.perf_counter()
            roots["c"] = T.beacon_state_root(cur, fork)
            c_ms.append((time.perf_counter() - t0) * 1e3)

        arms = [arm_a, arm_b, arm_c]
        for k in range(3):
            arms[(slot + k) % 3]()
        assert roots["a"] == roots["b"] == roots["c"], f"{fork} slot {slot}: the arms' roots differ"
    kernel = copy_kernel_ms(parent)
    ref = torch_copy_ms(int(np.median(live)))
    clone_med = float(np.median(clone_ms))
    kernel_med = float(np.median(kernel)) if kernel else None
    out = {
        "clone": stats(clone_ms),
        "clone_copy_kernel": stats(kernel) if kernel else "not measured",
        "clone_rest_median_ms": round(clone_med - kernel_med, 3) if kernel else "not measured",
        "live_bytes_median": int(np.median(live)), "device_bytes_median": int(np.median(held)),
        "torch_d2d_same_bytes": stats(ref),
        "a_clone_edit_root_release_per_slot": stats(a_ms), "b_linear_warm_per_slot": stats(b_ms),
        "c_restage_cold_per_slot": stats(c_ms),
        "validators_at_end": enc.length("validators"), "roots_equal_every_slot": True,
    }
    if kernel:
        out["copy_kernel_GBps"] = round(out["live_bytes_median"] / (kernel_med * 1e-3) / 1e9, 1)
    out["torch_d2d_GBps"] = round(out["live_bytes_median"] / (float(np.median(ref)) * 1e-3) / 1e9, 1)
    parent.release()
    lin.release()
    return out


def main():
    lighthouse_b200.init(0)
    import torch
    torch.cuda.init()
    res = {"card": card(), "slots": N_SLOTS, "n_validators": N_VALIDATORS}
    for fork, seed in (("deneb", 1), ("electra", 2)):
        res[fork] = run(fork, seed)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
