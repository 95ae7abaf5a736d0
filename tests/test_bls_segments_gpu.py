"""GPU: segmented passes, several independent batch checks in one device pass (lhb200_bls_batch_set_segments,
lhb200_verify_signature_set_batches), and the coalescing of concurrent lhb200_verify_signature_sets calls built on them.

Batch k of a pass must get exactly what verifying batch k alone with the same scalars gives: the same verdict, the same
per-set statuses and the same final-exponentiated product (lhb200_bls_batch_segment_gt against the C oracle run on
batch k alone).  A bad set in one batch must not touch the verdict of any other batch.
"""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from tests import oracle_lib as O
from oracle import bls_ref as B
from tests.test_bls_grouped_gpu import Ctx
from tests.test_bls_regimes_gpu import GT_ONE, EDGE_RANDS, V, _non_subgroup_g2, rotated

pytestmark = pytest.mark.gpu

# ragged segments, 1-set segments among them
SIZES = [1, 5, 64, 1, 17, 3, 128, 1, 30, 2]


@pytest.fixture(scope="module")
def ctx(gpu):
    from lighthouse_b200 import bls
    c = Ctx(bls)
    yield c
    c.table.destroy()


def offsets_of(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def distinct_batch(ctx, n, seed, keys=None):
    """n sets over n distinct messages, 1-3 keys each (a few of 128) -> (AttestationBatch, rands)"""
    rng = np.random.default_rng(seed)
    kc = rng.integers(1, 4, size=n) if keys is None else np.full(n, keys)
    if keys is None:
        kc[rng.choice(n, size=1 + n // 100, replace=False)] = 128
    ab, _, _, rands = ctx.batch(kc, np.arange(n), n, seed)
    return ab, rands


def segment(ab_sigs, msgs, pks, offs, rands, bo, k):
    """batch k of a segmented input, alone: (sigs, msgs, pks, offsets from 0, rands)"""
    lo, hi = int(bo[k]), int(bo[k + 1])
    k0, k1 = int(offs[lo]), int(offs[hi])
    return (ab_sigs[96 * lo:96 * hi], msgs[32 * lo:32 * hi], pks[96 * k0:96 * k1],
            (offs[lo:hi + 1] - k0).astype(np.uint32), rands[lo:hi])


def run_segments(bls, bo, n, n_keys, upload):
    b = bls.Batch(n, max(n_keys, 1))
    try:
        b.set_segments(bo)
        upload(b)
        b.enqueue()
        ok, st = b.segment_result(want_status=True)
        return ok, st.copy(), [b.segment_gt(k) for k in range(len(bo) - 1)], b.plan(), b.launches
    finally:
        b.destroy()


def test_segment_gt_matches_oracle_alone(ctx):
    """every segment's GT equals the oracle's for that segment alone (every set contributes: messages rotated inside
    each segment), with the edge scalars at segment ends; a valid input gives verdict 1 and GT one per segment"""
    bls = ctx.bls
    bo = offsets_of(SIZES)
    n, K = int(bo[-1]), len(SIZES)
    ab, rands = distinct_batch(ctx, n, 0x5E6)
    ends = sorted({int(x) for x in bo[:-1]} | {int(x) - 1 for x in bo[1:]})
    r = rands.copy()
    for j, i in enumerate(ends):
        r[i] = EDGE_RANDS[j % len(EDGE_RANDS)]
    nk = int(ab.offsets[-1])
    ok, st, gts, plan, _ = run_segments(bls, bo, n, nk, lambda b: b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, r))
    assert ok.all() and not st.any() and all(g == GT_ONE for g in gts)
    assert plan["segments"] == K and plan["sum"] == "k_g2_segment_sum" and plan["final"] == "k_final_segments"
    assert plan["miller"] == "k_miller_warp" and plan["groups"] == 0 and plan["fp12_reduce_levels"] == 0
    assert plan["sum_levels"] == 3   # the 128-set segment: 8, 64, 512
    msgs = b"".join(rotated(ab.msgs[32 * int(bo[k]):32 * int(bo[k + 1])], SIZES[k]) for k in range(K))
    want = [O.bls_verify_signature_sets(*segment(ab.sigs, msgs, ab.pks, ab.offsets, r, bo, k), want_gt=True)
            for k in range(K)]
    assert not any(w[0] for w in want) and all(w[1] != GT_ONE for w in want)
    idx = ab.committees.reshape(-1)
    uploads = {
        "explicit": lambda b: b.upload(ab.sigs, msgs, ab.pks, ab.offsets, r),
        "streamed": lambda b: b.upload_async(ab.sigs, msgs, ab.pks, ab.offsets, r),
        "indexed": lambda b: b.upload_indexed(ctx.table, ab.sigs, msgs, idx, ab.offsets, r),
    }
    for name, up in uploads.items():
        ok, st, gts, _, _ = run_segments(bls, bo, n, nk, up)
        assert not ok.any() and not st.any(), name
        for k in range(K):
            assert gts[k] == want[k][1], f"{name}: segment {k} ({SIZES[k]} sets): GT differs from the oracle alone"


def bad_input(ctx, n, bo, seg_all, seg_swap, seg_msg, seed):
    """statuses 1-6, a swapped signature pair and a wrong message in segment seg_all; only a swapped pair in seg_swap;
    only a wrong message in seg_msg -> (sigs, msgs, pks, offsets, rands)"""
    ab, rands = distinct_batch(ctx, n, seed)
    offs = ab.offsets
    comm = ab.committees.reshape(-1)
    sets_idx = [list(comm[offs[i]:offs[i + 1]]) for i in range(n)]
    sigs, msgs = bytearray(ab.sigs), bytearray(ab.msgs)
    bad_g2 = B.g2_compress(_non_subgroup_g2())

    def swap(i, j):
        si, sj = bytes(sigs[96 * i:96 * i + 96]), bytes(sigs[96 * j:96 * j + 96])
        sigs[96 * i:96 * i + 96], sigs[96 * j:96 * j + 96] = sj, si

    lo = int(bo[seg_all])
    s1 = bytes(sigs[96 * (lo + 1):96 * (lo + 2)])
    sigs[96 * lo:96 * lo + 96] = bytes(96)                                   # 1
    sigs[96 * (lo + 1):96 * (lo + 2)] = bytes([s1[0] & 0x7F]) + s1[1:]      # 2
    sigs[96 * (lo + 2):96 * (lo + 3)] = bad_g2                              # 3
    sets_idx[lo + 3] = []                                                   # 4
    sets_idx[lo + 4] = [0, V]                                               # 5: pk_0 + (-pk_0)
    sets_idx[lo + 5] = [sets_idx[lo + 5][0], V + 1]                         # 6: a malformed key
    swap(lo + 6, lo + 7)
    msgs[32 * (lo + 8):32 * (lo + 9)] = bytes(32)
    lo = int(bo[seg_swap])
    swap(lo, lo + 1)
    lo = int(bo[seg_msg])
    msgs[32 * lo:32 * lo + 32] = bytes([msgs[32 * lo] ^ 1]) + bytes(msgs[32 * lo + 1:32 * lo + 32])
    idx = np.array([j for s in sets_idx for j in s], dtype=np.uint32)
    new_offs = np.concatenate([[0], np.cumsum([len(s) for s in sets_idx])]).astype(np.uint32)
    bad_key = ctx.table_ext[1].copy()
    bad_key[0] |= 0x80
    pks = np.vstack([ctx.table_ext, bad_key[None]])[idx].tobytes()
    return bytes(sigs), bytes(msgs), pks, new_offs, rands


def test_isolation_of_bad_sets(ctx):
    """the segments holding bad sets fail, every other segment passes, and the statuses equal the oracle's, through the
    staged API and through lhb200_verify_signature_set_batches"""
    sizes = [12, 40, 9, 64, 1, 33, 2, 20]
    bo = offsets_of(sizes)
    n = int(bo[-1])
    sigs, msgs, pks, offs, rands = bad_input(ctx, n, bo, 1, 3, 5, 0x150)
    _, o_st = O.bls_verify_signature_sets(sigs, msgs, pks, offs, rands, want_status=True)
    assert sorted(set(o_st) - {0}) == [1, 2, 3, 4, 5, 6]
    want_ok = np.array([k not in (1, 3, 5) for k in range(len(sizes))])
    for k in range(len(sizes)):
        alone = O.bls_verify_signature_sets(*segment(sigs, msgs, pks, offs, rands, bo, k))
        assert alone == want_ok[k], k
    ok, st, _, _, _ = run_segments(ctx.bls, bo, n, int(offs[-1]), lambda b: b.upload(sigs, msgs, pks, offs, rands))
    np.testing.assert_array_equal(ok, want_ok)
    np.testing.assert_array_equal(st, o_st)
    for r in (rands, None):
        ok, st = ctx.bls.verify_signature_set_batches(sigs, msgs, pks, offs, bo, r, want_status=True)
        np.testing.assert_array_equal(ok, want_ok)
        np.testing.assert_array_equal(st, o_st)


SEGMENT_PROBE = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import lighthouse_b200
from lighthouse_b200 import bls
lighthouse_b200.init(0)
d = np.load(sys.argv[2])
bo, offs = d["bo"], d["offsets"]
b = bls.Batch(len(offs) - 1, max(int(offs[-1]), 1))
b.set_segments(bo)
b.upload(d["sigs"].tobytes(), d["msgs"].tobytes(), d["pks"].tobytes(), offs, d["rands"])
b.enqueue()
ok, st = b.segment_result(want_status=True)
print(json.dumps({"ok": ok.tolist(), "status": bytes(st).hex(), "plan": b.plan(),
                  "gt": [b.segment_gt(k).hex() for k in range(len(bo) - 1)]}))
"""


def test_grouping_stays_inside_segments(ctx, tmp_path):
    """segments that share messages with each other and within themselves: the groups never span two segments (the
    plan's group count is the sum of the per-segment counts), and the GT values, verdicts and statuses equal those of
    the same pass with LHB_GROUP_MESSAGES=0 and of the oracle on each segment alone"""
    rng = np.random.default_rng(0x6E7)
    sizes = [40, 1, 24, 64, 7]
    bo = offsets_of(sizes)
    n, m = int(bo[-1]), 6
    assign = rng.integers(0, m, size=n)
    ab, pool, assign, rands = ctx.batch(rng.integers(1, 4, size=n), assign, m, 0x6E7)
    msgs = b"".join(pool[(g + 1) % m] for g in assign)       # every set contributes
    per_seg = sum(len(set(assign[bo[k]:bo[k + 1]])) for k in range(len(sizes)))
    assert per_seg > m                                        # messages shared across segments
    ok, st, gts, plan, _ = run_segments(ctx.bls, bo, n, int(ab.offsets[-1]),
                                        lambda b: b.upload(ab.sigs, msgs, ab.pks, ab.offsets, rands))
    assert plan["groups"] == per_seg and plan["group_sum"] == "k_g1_group_sum", plan
    assert not ok.any() and not st.any()
    for k in range(len(sizes)):
        _, o_gt = O.bls_verify_signature_sets(*segment(ab.sigs, msgs, ab.pks, ab.offsets, rands, bo, k), want_gt=True)
        assert gts[k] == o_gt, k
    f = tmp_path / "seg.npz"
    np.savez(f, sigs=np.frombuffer(ab.sigs, np.uint8), msgs=np.frombuffer(msgs, np.uint8),
             pks=np.frombuffer(ab.pks, np.uint8), offsets=ab.offsets, rands=rands, bo=bo)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", SEGMENT_PROBE, root, str(f)], env=dict(os.environ, LHB_GROUP_MESSAGES="0"),
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    row = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert row["plan"]["groups"] == 0 and row["plan"]["segments"] == len(sizes)
    assert row["ok"] == ok.tolist() and row["status"] == bytes(st).hex()
    assert row["gt"] == [g.hex() for g in gts]


def test_pass_limit(ctx):
    """the largest input that fits one pass (sets + batches = 8 x SMs) runs as one pass; one more set makes two
    passes with the same verdicts and statuses; the staged form rejects the larger input"""
    from lighthouse_b200 import _ffi
    bls = ctx.bls
    limit = 8 * ctx.n_sm
    K = 8
    sizes = [(limit - K) // K] * K
    sizes[-1] += limit - K - sum(sizes)
    n = sum(sizes) + 1
    ab, rands = distinct_batch(ctx, n, 0x1A7, keys=1)
    msgs = bytearray(ab.msgs)
    msgs[32 * 5] ^= 1                                          # batch 0 fails
    msgs = bytes(msgs)
    one_pass_launches = None
    for big in (False, True):
        sz = sizes[:-1] + [sizes[-1] + big]
        bo = offsets_of(sz)
        m = int(bo[-1])
        want = [bls.verify_signature_sets_raw(*segment(ab.sigs, msgs, ab.pks, ab.offsets, rands, bo, k), want_status=True)
                for k in range(K)]
        offs = ab.offsets[:m + 1]
        l0 = _ffi.lib.lhb200_launch_count()
        ok, st = bls.verify_signature_set_batches(ab.sigs[:96 * m], msgs[:32 * m], ab.pks[:96 * m], offs, bo, rands[:m],
                                                  want_status=True)
        launches = _ffi.lib.lhb200_launch_count() - l0
        assert ok.tolist() == [w[0] for w in want] and ok.tolist() == [False] + [True] * (K - 1)
        np.testing.assert_array_equal(st, np.concatenate([w[1] for w in want]))
        if not big:
            one_pass = run_segments(bls, bo, m, m, lambda b: b.upload(ab.sigs[:96 * m], msgs[:32 * m], ab.pks[:96 * m],
                                                                      offs, rands[:m]))
            assert one_pass[3]["segments"] == K and one_pass[0].tolist() == ok.tolist()
            assert launches == one_pass[4], (launches, one_pass[4])
            one_pass_launches = launches
        else:
            assert launches > one_pass_launches
            b = bls.Batch(m, m)
            with pytest.raises(_ffi.Lhb200Error) as e:
                b.set_segments(bo)
            assert e.value.code == _ffi.EINVAL and "bls_batch_set_segments: " in str(e.value)
            b.destroy()


def test_argument_errors(ctx):
    from lighthouse_b200 import _ffi
    bls = ctx.bls
    ab, rands = distinct_batch(ctx, 6, 0xA26)
    ok, st = bls.verify_signature_set_batches(ab.sigs, ab.msgs, ab.pks, ab.offsets, [0, 3, 3, 6], rands, want_status=True)
    assert ok.tolist() == [True, False, True] and not st.any()        # an empty batch gives 0
    assert len(bls.verify_signature_set_batches(ab.sigs, ab.msgs, ab.pks, ab.offsets, [0], rands)) == 0
    bad = [([0, 4, 2, 6], rands, "batch offsets not monotone"),
           ([0, 3, 5], rands, "batch offsets do not span"),
           ([0, 3, 6], np.where(np.arange(6) == 4, 0, rands).astype(np.uint64), "zero random scalar")]
    for bo, r, msg in bad:
        with pytest.raises(_ffi.Lhb200Error) as e:
            bls.verify_signature_set_batches(ab.sigs, ab.msgs, ab.pks, ab.offsets, bo, r)
        assert e.value.code == _ffi.EINVAL and f"verify_signature_set_batches: {msg}" in str(e.value), str(e.value)
    b = bls.Batch(6, int(ab.offsets[-1]))
    for bo in ([0, 4, 2, 6], [0, 3, 3, 6], [1, 6]):
        with pytest.raises(_ffi.Lhb200Error) as e:
            b.set_segments(bo)
        assert e.value.code == _ffi.EINVAL and "bls_batch_set_segments: " in str(e.value)
    b.set_segments([0, 2, 6])
    with pytest.raises(_ffi.Lhb200Error) as e:                        # the upload must carry the segments' sets
        b.upload(ab.sigs[:96 * 5], ab.msgs[:32 * 5], ab.pks, ab.offsets[:6], rands[:5])
    assert e.value.code == _ffi.EINVAL
    b.destroy()


def test_concurrent_calls_are_coalesced(ctx):
    """32 threads (twice the passes the library keeps in flight, so calls queue) loop their own 64-set batches, some
    with a bad set, through the plugin call: every call gives its solo verdict and statuses, and fewer launches than
    solo calls would take prove that calls were merged; a lone call afterwards launches exactly what the staged path
    launches for the same batch"""
    from lighthouse_b200 import _ffi
    bls = ctx.bls
    T, ITERS = 32, 6
    batches = []
    for t in range(T):
        ab, _ = distinct_batch(ctx, 64, 0xC0A1 + t, keys=1 + (t % 3))
        sigs, msgs = bytearray(ab.sigs), bytearray(ab.msgs)
        if t % 4 == 1:
            sigs[96 * 7:96 * 8] = bytes(96)                       # status 1
        if t % 4 == 2:
            msgs[32 * 60] ^= 1                                    # wrong message: verdict 0, statuses 0
        batches.append((bytes(sigs), bytes(msgs), ab.pks, ab.offsets))
    solo, solo_launches = [], []
    for s, m, p, o in batches:
        l0 = _ffi.lib.lhb200_launch_count()
        solo.append(bls.verify_signature_sets_raw(s, m, p, o, want_status=True))
        solo_launches.append(_ffi.lib.lhb200_launch_count() - l0)
    assert [r[0] for r in solo] == [t % 4 not in (1, 2) for t in range(T)]
    errors = []

    def work(t):
        s, m, p, o = batches[t]
        for _ in range(ITERS):
            ok, st = bls.verify_signature_sets_raw(s, m, p, o, want_status=True)
            if ok != solo[t][0] or not np.array_equal(st, solo[t][1]):
                errors.append((t, ok, st))

    l0 = _ffi.lib.lhb200_launch_count()
    th = [threading.Thread(target=work, args=(t,)) for t in range(T)]
    [x.start() for x in th]
    [x.join() for x in th]
    launches = _ffi.lib.lhb200_launch_count() - l0
    assert not errors, errors[:3]
    assert launches < ITERS * sum(solo_launches), (launches, ITERS * sum(solo_launches))
    s, m, p, o = batches[0]
    l0 = _ffi.lib.lhb200_launch_count()
    assert bls.verify_signature_sets_raw(s, m, p, o)
    lone = _ffi.lib.lhb200_launch_count() - l0
    b = bls.Batch(64, int(o[-1]))
    b.upload_async(s, m, p, o)
    l0 = _ffi.lib.lhb200_launch_count()
    b.enqueue()
    assert b.result()
    assert lone == _ffi.lib.lhb200_launch_count() - l0 == b.launches
    b.destroy()
