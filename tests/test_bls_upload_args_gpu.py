"""Argument checks of the three host uploads of a batch handle (lhb200_bls_batch_upload, _upload_async,
_upload_indexed): every malformed input is rejected with LHB200_EINVAL and a message naming the entry point, and the
same handle then still verifies a valid batch."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, MAX_KEYS = 4, 4                                  # the handle holds exactly the valid batch: 4 sets of one key


@pytest.fixture(scope="module")
def valid(gpu):
    from lighthouse_b200 import bls
    sks = b"".join((i + 1).to_bytes(32, "big") for i in range(N + 1))
    _, pk96 = bls.sk_to_pk(sks)
    msgs = b"".join(hashlib.sha256(b"upload-args %d" % i).digest() for i in range(N))
    sigs = bls.sign(sks[:32 * N], msgs)
    table = bls.PubkeyTable(N + 1)
    table.append(pk96)
    yield dict(sigs=sigs, msgs=msgs, pks=pk96, offsets=np.arange(N + 1, dtype=np.uint32),
               rands=np.arange(1, N + 1, dtype=np.uint64), table=table)
    table.destroy()


def upload(kind, b, v, **over):
    a = dict(v, **over)
    if kind == "upload":
        b.upload(a["sigs"], a["msgs"], a["pks"], a["offsets"], a["rands"])
    elif kind == "upload_async":
        b.upload_async(a["sigs"], a["msgs"], a["pks"], a["offsets"], a["rands"])
    else:
        b.upload_indexed(a["table"], a["sigs"], a["msgs"], np.arange(a["offsets"][-1], dtype=np.uint32), a["offsets"],
                         a["rands"])


def null_indices(b, v):
    """lhb200_bls_batch_upload_indexed with keys in the offsets but no key indices"""
    from lighthouse_b200._ffi import lib, check, buf
    (ps, k1), (pm, k2) = buf(v["sigs"]), buf(v["msgs"])
    check(lib.lhb200_bls_batch_upload_indexed(b._h, v["table"]._h, ps, pm, None, v["offsets"].ctypes.data,
                                              v["rands"].ctypes.data, N), "lhb200_bls_batch_upload_indexed")


def bad_inputs(kind, v):
    """(words of the expected message, callable(batch)) for every malformed input of this upload; consecutive cases
    expect different messages, so a rejection that leaves the previous message in place fails"""
    zero_rands = v["rands"].copy()
    zero_rands[2] = 0
    cases = [
        ("bad arguments", lambda b: upload(kind, b, v, offsets=np.zeros(1, dtype=np.uint32))),       # no sets
        ("not monotone", lambda b: upload(kind, b, v, offsets=np.array([0, 2, 1, 3, 4], dtype=np.uint32))),
        ("bad arguments", lambda b: upload(kind, b, v, sigs=v["sigs"] + v["sigs"][:96],              # > max_sets
                                           msgs=v["msgs"] + v["msgs"][:32], offsets=np.arange(N + 2, dtype=np.uint32),
                                           rands=np.arange(1, N + 2, dtype=np.uint64))),
        ("zero random scalar", lambda b: upload(kind, b, v, rands=zero_rands)),
    ]
    if kind == "upload_indexed":
        cases.append(("no keys", lambda b: null_indices(b, v)))
    else:   # 5 keys, max_keys 4
        cases.append(("more keys", lambda b: upload(kind, b, v, offsets=np.array([0, 1, 2, 3, 5], dtype=np.uint32))))
    return cases


@pytest.mark.parametrize("kind", ["upload", "upload_async", "upload_indexed"])
def test_rejected_uploads_leave_the_handle_usable(valid, kind):
    from lighthouse_b200 import bls
    from lighthouse_b200._ffi import lib, EINVAL, Lhb200Error
    b = bls.Batch(N, MAX_KEYS)
    try:
        for reason, call in bad_inputs(kind, valid):
            with pytest.raises(Lhb200Error) as e:
                call(b)
            assert e.value.code == EINVAL, (kind, reason, str(e.value))
            msg = lib.lhb200_last_error().decode()
            assert msg.startswith(f"bls_batch_{kind}: ") and reason in msg, (kind, reason, msg)
            upload(kind, b, valid)
            b.enqueue()
            ok, st = b.result(want_status=True)
            assert ok is True and not st.any(), (kind, reason)
    finally:
        b.destroy()
