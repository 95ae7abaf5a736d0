"""Times lhb200_beacon_block_roots end to end (host buffers in and out, one call per batch) for Electra and Deneb blocks,
with every result checked against the generic from-spec merkleization of tests/ssz_spec.py in the same run.  Prints the
card and its power limit, then one JSON line per workload."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lighthouse_b200  # noqa: E402
from lighthouse_b200 import _ffi, ssz_schema as S, synthetic  # noqa: E402
from lighthouse_b200.tree_hash import FORKS  # noqa: E402
from tests import ssz_spec  # noqa: E402

MIN_SECONDS = 1.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def workloads():
    electra = lambda i, **kw: synthetic.beacon_block_electra(seed=300 + i, **kw)
    deneb = lambda i: synthetic.beacon_block_deneb(seed=300 + i)
    # mainnet-like Electra: 8 attestations over 8 committees of ~500 (a 1M-validator set), a handful of deposit requests
    mainnet = dict(committees_per_attestation=8, bits_per_committee=500, n_deposit_requests=4)
    return [("electra", "electra 1 block", [electra(0, **mainnet)]),
            ("electra", "electra 1 block, 8192 deposit requests", [electra(1, **dict(mainnet, n_deposit_requests=8192))]),
            # either side of the switch from container ops to the record kernel (more than 64 deposit requests)
            ("electra", "electra 1 block, 64 deposit requests", [electra(2, **dict(mainnet, n_deposit_requests=64))]),
            ("electra", "electra 1 block, 128 deposit requests", [electra(3, **dict(mainnet, n_deposit_requests=128))]),
            ("electra", "electra 32 blocks", [electra(i, **mainnet) for i in range(32)]),
            ("electra", "electra 32 blocks, 128 deposit requests each",
             [electra(i, **dict(mainnet, n_deposit_requests=128)) for i in range(32)]),
            ("deneb", "deneb 1 block", [deneb(0)]),
            ("deneb", "deneb 32 blocks", [deneb(i) for i in range(32)])]


def main():
    lighthouse_b200.init(0)
    print(json.dumps({"card": card(), "library": _ffi.LIB_PATH}))
    lib = _ffi.lib
    for fork, label, blocks in workloads():
        typ = S.BEACON_BLOCK_BY_FORK[fork]
        want = b"".join(ssz_spec.hash_tree_root(typ, v) for v, _ in blocks)
        blob = b"".join(b for _, b in blocks)
        n = len(blocks)
        offs = (C.c_uint64 * (n + 1))()
        for i, (_, b) in enumerate(blocks):
            offs[i + 1] = offs[i] + len(b)
        src = C.create_string_buffer(blob, len(blob))
        out = C.create_string_buffer(32 * n)

        def call():
            rc = lib.lhb200_beacon_block_roots(src, C.cast(offs, C.c_void_p), n, FORKS[fork], 0, out, None)
            assert rc == 0, (rc, lib.lhb200_last_error())

        for _ in range(5):
            call()
        assert out.raw == want, label
        times = []
        t_end = time.perf_counter() + MIN_SECONDS
        while time.perf_counter() < t_end or len(times) < 10:
            t = time.perf_counter()
            call()
            times.append(time.perf_counter() - t)
        assert out.raw == want, label
        times.sort()
        print(json.dumps({"workload": label, "blocks": n, "bytes": len(blob), "calls": len(times),
                          "ms_per_call_mean": round(1e3 * sum(times) / len(times), 4),
                          "ms_per_call_median": round(1e3 * times[len(times) // 2], 4),
                          "us_per_block_mean": round(1e6 * sum(times) / len(times) / n, 2), "match_ssz_spec": True}))


if __name__ == "__main__":
    main()
