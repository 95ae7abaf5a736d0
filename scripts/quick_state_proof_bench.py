"""Merkle proofs by generalized index from resident BeaconStates and BeaconBlock bodies (lhb200_state_proofs,
lhb200_beacon_block_body_proofs).  Prints one JSON line with the card name and power limit read in the same run.

Arms, 500 000 validators, converted Deneb and Electra handles on the 64-slot synthetic chain of
quick_warm_chain_bench.py (two handles, one a clone of the other, take the same edits):
  chain_triple       per slot: edits + the light-client triple (finalized root, both sync committees) in one call
  chain_root         per slot: edits + lhb200_state_root alone
  triple_rooted      the triple on a handle with nothing pending
  validators_<n>     n = 1 000 and 100 000 validator proofs on the incremental handle and on a cold (staged,
                     non-incremental) one: call time, gather-kernel time from CUDA events, proofs/s
  blobs_<n>          the six blob inclusion proofs of each of n = 1 and 32 Electra blocks, against
                     lhb200_beacon_block_roots on the same blocks
Every branch of the run is verified against its root: state triples with hashlib (each node read back as the first
sibling of its own sibling's branch), validator proofs through lhb200_verify_merkle_proofs, blob proofs with hashlib."""
import ctypes as C
import hashlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import _ffi, tree_hash as T
from lighthouse_b200.synthetic import beacon_block_electra, beacon_state_deneb_ssz
from quick_warm_chain_bench import N_SLOTS, N_VALIDATORS, Encoding, card, slot_work, stats


def h(a, b):
    return hashlib.sha256(a + b).digest()


def fold(leaf, branch, g):
    for k, sib in enumerate(branch):
        leaf = h(sib, leaf) if (g >> k) & 1 else h(leaf, sib)
    return leaf


def triple(fork):
    if fork == "electra":
        return [T.FINALIZED_ROOT_INDEX_ELECTRA, T.CURRENT_SYNC_COMMITTEE_INDEX_ELECTRA, T.NEXT_SYNC_COMMITTEE_INDEX_ELECTRA]
    return [T.FINALIZED_ROOT_INDEX, T.CURRENT_SYNC_COMMITTEE_INDEX, T.NEXT_SYNC_COMMITTEE_INDEX]


def verify_state_branches(st, gis, root, branches):
    """Each node is the first sibling of its sibling's branch (one more call, nothing pending: same root)."""
    r2, sib = st.proofs([g ^ 1 for g in gis])
    assert r2 == root
    for g, b, s in zip(gis, branches, sib):
        assert fold(s[0], b, g) == root, g


def verify_validator_proofs(flat, gis, depth, leaves, root):
    n = len(gis)
    idx = np.ascontiguousarray(gis - np.uint64(1 << depth))
    ok = C.create_string_buffer(n)
    p_l, k1 = _ffi.buf(leaves)
    p_r, k2 = _ffi.buf(root * n)
    _ffi.check(_ffi.lib.lhb200_verify_merkle_proofs(p_l, flat.ctypes.data, depth, idx.ctypes.data, p_r, n, ok),
               "lhb200_verify_merkle_proofs")
    assert ok.raw == b"\x01" * n


def validator_arm(st, enc, fork, reps=10):
    nv = enc.length("validators")
    leaves = T.validator_roots(bytes(enc.parts["validators"]))
    top = 64 if fork == "electra" else 32          # leaves of the state's top tree
    depth = top.bit_length() - 1 + 1 + 40          # top tree, length mix-in, List[Validator, 2^40]
    g0 = (2 * (top + 11)) << 40
    out = {}
    rng = np.random.default_rng(3)
    for n in (1000, 100_000):
        gis = np.ascontiguousarray(np.sort(rng.choice(nv, size=n, replace=False)).astype(np.uint64) + np.uint64(g0))
        call, gather = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            root, flat = st.proofs(gis, raw=True)
            call.append((time.perf_counter() - t0) * 1e3)
            gather.append(T.debug_proof_gather_ms())
        sel = (gis - np.uint64(g0)).astype(np.int64)
        lv = b"".join(leaves[32 * i: 32 * i + 32] for i in sel.tolist())
        verify_validator_proofs(flat, gis, depth, lv, root)
        g = float(np.median(gather))
        out[f"validators_{n}"] = {"call": stats(call), "gather_kernel": stats(gather),
                                  "proofs_per_s_call": round(n / (float(np.median(call)) / 1e3)),
                                  "proofs_per_s_gather": round(n / (g / 1e3)) if g > 0 else None}
    return out


def run_chain(fork, seed):
    rng = np.random.default_rng(seed)
    ssz = beacon_state_deneb_ssz(N_VALIDATORS, seed=seed, fork=fork, n_votes=3, n_summaries=40)
    enc = Encoding(ssz, fork)
    a = T.ResidentState(ssz, fork)
    a.enable_incremental()
    a.root()
    gis = triple(fork)
    t_triple, t_root = [], []
    b = None
    for slot in range(N_SLOTS):
        patches, edits, hdr = slot_work(rng, enc, fork, slot)
        if b is None:   # converted by the first edits, then cloned: both handles follow the same chain
            a.patch_batch(patches)
            a.list_edit(edits)
            a.set_payload_header(hdr)
            a.root()
            b = a.clone()
            continue
        for st in (a, b) if slot % 2 else (b, a):
            t0 = time.perf_counter()
            st.patch_batch(patches)
            st.list_edit(edits)
            st.set_payload_header(hdr)
            if st is a:
                root_a, branches = a.proofs(gis)
                t_triple.append((time.perf_counter() - t0) * 1e3)
            else:
                root_b = b.root()
                t_root.append((time.perf_counter() - t0) * 1e3)
        assert root_a == root_b, f"{fork} slot {slot}: proof root differs from lhb200_state_root"
        verify_state_branches(a, gis, root_a, branches)
    rooted = []
    for _ in range(50):
        t0 = time.perf_counter()
        root, branches = a.proofs(gis)
        rooted.append((time.perf_counter() - t0) * 1e3)
    verify_state_branches(a, gis, root, branches)
    out = {"chain_triple_per_slot": stats(t_triple), "chain_root_per_slot": stats(t_root), "triple_rooted": stats(rooted)}
    out["incremental"] = validator_arm(a, enc, fork)
    b.release()
    a.release()
    cold = T.ResidentState(enc.ssz(), fork)
    out["cold"] = validator_arm(cold, enc, fork, reps=5)
    cold.release()
    return out


def run_blobs():
    blocks = [beacon_block_electra(seed=200 + i, n_blobs=6)[1] for i in range(32)]
    body_t_commitments = [beacon_block_electra(seed=200 + i, n_blobs=6)[0]["body"]["blob_kzg_commitments"] for i in range(32)]
    out = {}
    for n in (1, 32):
        proofs = [(b, T.kzg_commitment_gindex(j)) for b in range(n) for j in range(6)]
        tp, tr = [], []
        for _ in range(30):
            t0 = time.perf_counter()
            body_roots, branches = T.beacon_block_body_proofs(blocks[:n], proofs, "electra")
            tp.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            _, body2 = T.beacon_block_roots(blocks[:n], "electra", want_body_roots=True)
            tr.append((time.perf_counter() - t0) * 1e3)
        assert body_roots == body2
        for (b, g), br in zip(proofs, branches):
            c = body_t_commitments[b][g - 54 * 4096]
            assert len(br) == 17 and fold(h(c[:32], c[32:] + bytes(16)), br, g) == body_roots[b]
        out[f"blobs_{n}_blocks"] = {"body_proofs": stats(tp), "block_roots": stats(tr)}
    return out


def main():
    lighthouse_b200.init(0)
    res = {"card": card(), "slots": N_SLOTS, "n_validators": N_VALIDATORS}
    for fork, seed in (("deneb", 1), ("electra", 2)):
        res[fork] = run_chain(fork, seed)
    res.update(run_blobs())
    res["every_branch_verified"] = True
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
