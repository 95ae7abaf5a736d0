"""GPU: every device point decoder against the encoding reference (tests/bls_encoding_spec.py), status by status.

Each decode site of the library gets the whole corpus of its encoding: the batch entry points (lhb200_g1_decompress_validate,
lhb200_g1_deserialize_uncompressed, lhb200_g2_decompress with n > 1), the aggregations and the pubkey table (one call
per corpus entry next to a valid point), and the batch verifier, where the corpus entries sit first, in the middle,
last and in between valid sets: the signature stage in warp and in lane mode, the key stage in its split, per-set and
TMA kernels.  Each batch asserts the kernel that ran (lhb200_bls_batch_plan) instead of assuming it from the size.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bls_ref as B
from tests import bls_encoding_spec as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NK = 64                                  # distinct signing keys of the valid sets


class Keys:
    def __init__(self, bls):
        from lighthouse_b200 import _ffi
        self.bls, self.ffi = bls, _ffi
        self.sks = [B.interop_secret_key(i) for i in range(NK)]
        _, pk96 = bls.sk_to_pk(b"".join(s.to_bytes(32, "big") for s in self.sks))
        self.pk96 = [pk96[96 * i:96 * i + 96] for i in range(NK)]
        self.pts = [S.decode_g1_uncompressed(k)[1] for k in self.pk96]
        self.n_sm = run_batch(bls, *self.batch([1]))[2]["n_sm"]

    def batch(self, sizes, n=1, seed=0):
        """n valid sets of len(sizes)-cycled key counts, distinct messages -> (sigs, msgs, key lists, offsets, rands)"""
        rng = np.random.default_rng(seed)
        keys, sks, msgs = [], [], []
        for i in range(n):
            idx = [(7 * i + 3 * j) % NK for j in range(sizes[i % len(sizes)])]
            keys.append([self.pk96[j] for j in idx])
            sks.append(sum(self.sks[j] for j in idx) % B.R)
            msgs.append(hashlib.sha256(b"enc%d/%d" % (seed, i)).digest())
        sigs = self.bls.sign(b"".join(s.to_bytes(32, "big") for s in sks), b"".join(msgs))
        rands = rng.integers(1, 2 ** 64 - 1, size=n, dtype=np.uint64, endpoint=True)
        return bytearray(sigs), b"".join(msgs), keys, rands


def flatten(keys):
    offs = np.concatenate([[0], np.cumsum([len(k) for k in keys])]).astype(np.uint32)
    return b"".join(b"".join(k) for k in keys), offs


def run_batch(bls, sigs, msgs, keys, rands):
    pks, offs = flatten(keys)
    n = len(keys)
    b = bls.Batch(n, max(len(pks) // 96, 1))
    try:
        b.upload(bytes(sigs), msgs, pks, offs, rands)
        b.enqueue()
        ok, st = b.result(want_status=True)
        return ok, st.copy(), b.plan()
    finally:
        b.destroy()


def spread(m, n):
    """m distinct set positions in [0, n): 0, n // 2 and n - 1 first, the rest evenly in between"""
    assert m + 3 <= n
    ends = [0, n // 2, n - 1]
    rest = [p for p in np.unique(np.linspace(1, n - 2, 2 * m).round().astype(int)) if p not in ends]
    step = len(rest) / (m - 3) if m > 3 else 1
    return (ends + [int(rest[int(k * step)]) for k in range(m - 3)])[:m]


@pytest.fixture(scope="module")
def K(gpu):
    from lighthouse_b200 import bls
    return Keys(bls)


# ---- single-call entry points -------------------------------------------------------------------------------------
def test_g1_decompress_validate(K):
    """lhb200_g1_decompress_validate (PublicKey::deserialize) on the whole 48-byte corpus in one call"""
    items = S.corpora()["g1c"]
    out, st = K.bls.decompress_validate_pubkeys(b"".join(b for _, b, _ in items))
    for i, (name, b, o) in enumerate(items):
        assert st[i] == S.G1_DECOMPRESS_VALIDATE[o], (name, int(st[i]), o)
        want = B.g1_uncompressed(S.decode_g1_compressed(b)[1]) if o == S.OK else bytes(96)
        assert out[96 * i:96 * i + 96] == want, name


def test_g1_deserialize_uncompressed(K):
    """lhb200_g1_deserialize_uncompressed (k_g1_load_points) on the whole 96-byte key corpus in one call"""
    items = S.corpora()["g1u"]
    n = len(items)
    pk48 = np.zeros(48 * n, dtype=np.uint8)
    st = np.zeros(n, dtype=np.uint8)
    p, keep = K.ffi.buf(b"".join(b for _, b, _ in items))
    K.ffi.check(K.ffi.lib.lhb200_g1_deserialize_uncompressed(p, n, pk48.ctypes.data, st.ctypes.data), "deserialize")
    for i, (name, b, o) in enumerate(items):
        assert st[i] == S.G1_DESERIALIZE_UNCOMPRESSED[o], (name, int(st[i]), o)
        want = B.g1_compress(S.decode_g1_uncompressed(b)[1]) if o == S.OK else bytes(48)
        assert pk48[48 * i:48 * i + 48].tobytes() == want, name


def test_g2_decompress_batch(K):
    """lhb200_g2_decompress (Signature::deserialize) with n > 1 through the C ABI: statuses and the 192-byte affine
    output (x.c1 | x.c0 | y.c1 | y.c0) of every accepted encoding"""
    items = S.corpora()["g2c"]
    n = len(items)
    out = C.create_string_buffer(192 * n)
    st = C.create_string_buffer(n)
    p, keep = K.ffi.buf(b"".join(b for _, b, _ in items))
    K.ffi.check(K.ffi.lib.lhb200_g2_decompress(p, n, out, st), "lhb200_g2_decompress")
    for i, (name, b, o) in enumerate(items):
        assert st.raw[i] == S.G2_DECOMPRESS[o], (name, st.raw[i], o)
        got = out.raw[192 * i:192 * i + 192]
        if st.raw[i] == 0:
            (x0, x1), (y0, y1) = S.decode_g2_compressed(b)[1]
            assert got == b"".join(v.to_bytes(48, "big") for v in (x1, x0, y1, y0)), name
        else:
            assert got == (bytes([0x40]) + bytes(191) if st.raw[i] == 1 else bytes(192)), name


def test_g1_aggregate_and_pubkey_table(K):
    """lhb200_g1_aggregate and PubkeyTable.append (k_g1_load_points, k_table_import): each corpus key after a valid
    key.  The aggregate refuses malformed and off-curve keys and adds the rest (infinity is the identity); the table
    refuses every call with a key that is not a finite curve point, and then holds nothing"""
    bls, ffi = K.bls, K.ffi
    for name, b, o in S.corpora()["g1u"]:
        o48, o96 = C.create_string_buffer(48), C.create_string_buffer(96)
        p, keep = ffi.buf(K.pk96[5] + b)
        rc = ffi.lib.lhb200_g1_aggregate(p, 2, o48, o96)
        if S.g1_aggregate_refused(b):
            assert rc == ffi.EDECODE, (name, rc)
        else:
            assert rc == 0, (name, rc)
            want = B.g1_add(K.pts[5], S.decode_g1_uncompressed(b)[1])
            assert o96.raw == B.g1_uncompressed(want) and o48.raw == B.g1_compress(want), name
        t = bls.PubkeyTable(2)
        try:
            if S.table_append_refused(b):
                with pytest.raises(ffi.Lhb200Error) as e:
                    t.append(K.pk96[5] + b)
                assert e.value.code == ffi.EDECODE and len(t) == 0, name
            else:
                t.append(K.pk96[5] + b)
                assert len(t) == 2, name
        finally:
            t.destroy()


def test_g2_aggregate(K):
    """lhb200_g2_aggregate (k_g2_load_points): each corpus signature after a valid one; refused iff malformed or off
    the curve, otherwise the sum (no subgroup check: aggregation takes checked signatures)"""
    base = bytes(K.batch([1])[0][:96])
    base_pt = S.decode_g2_compressed(base)[1]
    for name, b, o in S.corpora()["g2c"]:
        out = C.create_string_buffer(96)
        p, keep = K.ffi.buf(base + b)
        rc = K.ffi.lib.lhb200_g2_aggregate(p, 2, out)
        if S.g2_aggregate_refused(b):
            assert rc == K.ffi.EDECODE, (name, rc)
        else:
            assert rc == 0, (name, rc)
            assert out.raw == B.g2_compress(B.g2_add(base_pt, S.decode_g2_compressed(b)[1])), name


# ---- the batch verifier -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["warp", "lane"])
def test_signature_decoding_in_batches(K, mode):
    """the signature corpus in one batch of valid sets: k_sig_prepare_warp (<= 6 sets per SM) or k_sig_prepare; each
    corpus set gets the reference's SET_* code, every other set keeps 0"""
    n = 6 * K.n_sm + (mode == "lane")
    items = S.corpora()["g2c"]
    if mode == "lane":
        items = items[::-1]                       # other entries at the ends
    sigs, msgs, keys, rands = K.batch([1], n, seed=n)
    ok, st, plan = run_batch(K.bls, sigs, msgs, keys, rands)
    assert ok and not st.any(), "the uncorrupted batch must verify"
    want = np.zeros(n, dtype=np.uint8)
    for (name, b, o), i in zip(items, spread(len(items), n)):
        sigs[96 * i:96 * i + 96] = b
        want[i] = S.SET_SIG[o]
    ok, st, plan = run_batch(K.bls, sigs, msgs, keys, rands)
    assert plan["sig"] == ("k_sig_prepare_warp" if mode == "warp" else "k_sig_prepare"), plan
    bad = [(items[k][0], int(st[i]), int(want[i])) for k, i in enumerate(spread(len(items), n)) if st[i] != want[i]]
    assert not bad and np.array_equal(st, want), bad[:10]
    assert ok is False


def key_corpus_batch(K, sizes, n_valid_between, seed):
    """valid sets with a corpus key in between every n_valid_between of them: the corpus key of entry k replaces key
    k mod (set size) of a set of sizes[k mod len(sizes)] keys -> (sigs, msgs, keys, rands, expected statuses, names)"""
    items = S.corpora()["g1u"]
    n = len(items) * (n_valid_between + 1) + 3
    sizes_of = [1] * n
    pos = spread(len(items), n)
    for k, i in enumerate(pos):   # the infinity key alone in its set: the aggregate key is at infinity (SET 5)
        sizes_of[i] = 1 if items[k][2] == S.INFINITY else sizes[k % len(sizes)]
    sigs, msgs, keys, rands = K.batch(sizes_of, n, seed=seed)
    want = np.zeros(n, dtype=np.uint8)
    names = {}
    for k, ((name, b, o), i) in enumerate(zip(items, pos)):
        j = (k // len(sizes)) % len(keys[i])
        keys[i][j] = b
        want[i] = S.batch_key_set_status(keys[i])
        names[i] = f"{name} (key {j} of {len(keys[i])})"
    return sigs, msgs, keys, rands, want, names


@pytest.mark.parametrize("kernel", ["k_pk_partial+k_pk_combine", "k_pk_aggregate"])
def test_key_decoding_in_batches(K, kernel):
    """the 96-byte key corpus inside sets of 1 to 17 keys (every slice of the split kernel), between valid sets; the
    per-set kernel runs above 8192 sets"""
    if kernel == "k_pk_aggregate":
        sigs, msgs, keys, rands, want, names = key_corpus_batch(K, [1, 2, 3, 5, 9, 17], 39, seed=2)
        assert len(keys) > 8192
    else:
        sigs, msgs, keys, rands, want, names = key_corpus_batch(K, [1, 2, 3, 5, 9, 17], 1, seed=1)
    ok, st, plan = run_batch(K.bls, sigs, msgs, keys, rands)
    assert plan["key"] == kernel, plan
    bad = [(names.get(i), int(st[i]), int(want[i])) for i in np.nonzero(st != want)[0]]
    assert not bad, bad[:10]
    assert set(np.unique(want)) == {0, 5, 6} and ok is False


def test_key_decoding_in_the_tma_kernel(K, tmp_path):
    """k_pk_aggregate_tma (selected at start-up by LHB_PK_TMA=1, so in a subprocess through scripts/regime_probe.py)
    decodes keys from 32-bit words of its shared-memory ring with its own flag masks: corpus keys in both halves of a
    two-key slot and in the last, partial stage of 3- and 5-key sets"""
    sigs, msgs, keys, rands, want, names = key_corpus_batch(K, [3, 5], 1, seed=3)
    pks, offs = flatten(keys)
    f = tmp_path / "tma_keys.npz"
    np.savez(f, sigs=np.frombuffer(bytes(sigs), np.uint8), msgs=np.frombuffer(msgs, np.uint8),
             pks=np.frombuffer(pks, np.uint8), offsets=offs, rands=rands)
    slots = {int(n.split("key ")[1].split(" ")[0]) for n in names.values()}
    assert slots == {0, 1, 2, 3, 4}
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "regime_probe.py"), str(f)],
                         env=dict(os.environ, LHB_PK_TMA="1"), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    row = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")][0]
    assert row["plan"]["key"] == "k_pk_aggregate_tma", row["plan"]
    st = np.frombuffer(bytes.fromhex(row["status"]), dtype=np.uint8)
    bad = [(names.get(i), int(st[i]), int(want[i])) for i in np.nonzero(st != want)[0]]
    assert not bad, bad[:10]
    assert row["ok"] is False
