"""Runs the batches stored in .npz files through the batch verifier and prints one JSON line per file: verdict, per-set
statuses, GT bytes (the final-exponentiated product) and the kernel plan the library chose.  The kernel-selection
switches (LHB_G2_WARP, LHB_MILLER_WARP, LHB_MILLER_COOP, LHB_FINAL_WARP, LHB_PK_TMA) are read once per process, so
tests/test_bls_regimes_gpu.py runs this script once per switch set and compares the output with the oracle.

A file holds sigs, msgs, pks (uint8), offsets (uint32), rands (uint64) and optionally indices (uint32) + table
(uint8[T, 96]): with indices the keys come from a device pubkey table (upload_indexed), without them from the explicit
key buffer (upload, or upload_async when the file has async=1).

    python scripts/regime_probe.py a.npz [b.npz ...]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lighthouse_b200
from lighthouse_b200 import bls


def run(path):
    z = np.load(path)
    n = len(z["offsets"]) - 1
    b = bls.Batch(n, max(int(z["offsets"][-1]), 1))
    table = None
    try:
        if "indices" in z:
            table = bls.PubkeyTable(len(z["table"]))
            table.append(z["table"].tobytes())
            b.upload_indexed(table, z["sigs"], z["msgs"], z["indices"], z["offsets"], z["rands"])
        elif "async" in z and int(z["async"]):
            b.upload_async(z["sigs"], z["msgs"], z["pks"], z["offsets"], z["rands"])
        else:
            b.upload(z["sigs"], z["msgs"], z["pks"], z["offsets"], z["rands"])
        b.enqueue()
        ok, st = b.result(want_status=True)
        return {"file": os.path.basename(path), "n": n, "ok": bool(ok), "status": bytes(st).hex(),
                "gt": b.gt_bytes().hex() if not st.any() else None, "plan": b.plan()}
    finally:
        b.destroy()
        if table is not None:
            table.destroy()


if __name__ == "__main__":
    lighthouse_b200.init(0)
    for p in sys.argv[1:]:
        print(json.dumps(run(p)), flush=True)
