"""GPU: batches whose signature sets share messages.  The host uploads group the sets by message and the verifier
pairs each distinct message once, through the per-message sum of r_i apk_i (k_g1_group_sum).  The verdict, the per-set
statuses and the GT value (lhb200_bls_batch_gt) must equal the C oracle's, which pairs every set on its own.

The group counts straddle every seam where the hash, Miller and product-tree kernels switch (those stages are chosen
from the number of distinct messages), with three sets per group and one group holding a third of the batch (the
signature and key stages are chosen from the number of sets).  Each size runs a valid batch (GT one) and an "every group
contributes" batch: sets signed over pool[g] are verified against pool[g + 1 mod k], so no pair is trivial.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import oracle_lib as O
from oracle import bls_ref as B
from tests.test_bls_regimes_gpu import GT_ONE, EDGE_RANDS, MIX, V, _non_subgroup_g2, check_plan, run_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# group counts from the SM count s: both sides of every hash / Miller / product-tree switch
GROUP_SEAMS = [
    ("one_group", lambda s: 1), ("two_groups", lambda s: 2),
    ("miller_warp_4wpb_last", lambda s: 255), ("miller_warp_8wpb_first", lambda s: 256),
    ("miller_warp_no_reduce_last", lambda s: 511), ("miller_warp_reduce_first", lambda s: 512),
    ("hash_warp_last", lambda s: 6 * s), ("hash_pair_first", lambda s: 6 * s + 1),
    ("miller_warp_last", lambda s: 8 * s - 1), ("miller_coop_first", lambda s: 8 * s),
    ("hash_pair_last", lambda s: 4096), ("hash_lane_first", lambda s: 4097),
    ("coop_few_warps_last", lambda s: 7679), ("coop_full_first", lambda s: 7680),
]


def want_plan(n, m, s):
    """kernels the default switches choose for n sets over m distinct messages on s SMs"""
    return dict(
        groups=m, group_sum="k_g1_group_sum",
        sig="k_sig_prepare_warp" if n <= 6 * s else "k_sig_prepare",
        key="k_pk_partial+k_pk_combine" if n <= 8192 else "k_pk_aggregate",
        hash="k_hash_to_g2_warp" if m <= 6 * s else "k_hash_to_g2_pair" if m <= 4096 else "k_hash_to_g2",
        miller="k_miller_warp" if m + 1 <= 8 * s else "k_miller_coop")


def tree_levels(largest):
    levels = 1
    while 8 ** levels < largest:
        levels += 1
    return levels


def flip(msg):
    return bytes([msg[0] ^ 1]) + msg[1:]


class Ctx:
    def __init__(self, bls):
        from lighthouse_b200.synthetic import interop_pubkey_table
        self.bls = bls
        self.table96 = interop_pubkey_table(V)
        neg0 = self.table96[0].copy()                          # -pk_0
        y = B.P - int.from_bytes(neg0[48:].tobytes(), "big")
        neg0[48:] = np.frombuffer(y.to_bytes(48, "big"), dtype=np.uint8)
        self.table_ext = np.vstack([self.table96, neg0[None]])
        self.table = bls.PubkeyTable(V + 1)
        self.table.append(self.table_ext.tobytes())
        b = bls.Batch(1, 1)
        b.upload(bytes(96), bytes(32), self.table96[0].tobytes(), np.array([0, 1]), [1])
        b.enqueue(); b.result()
        self.n_sm = b.plan()["n_sm"]
        b.destroy()
        self.oracle_sets = 0
        O.set_threads(O.hw_threads())

    def batch(self, key_counts, assign, k, seed):
        """sets with the given key counts, set i signed over pool[assign[i]] (k random messages) ->
        (AttestationBatch, pool, assign, rands)"""
        from lighthouse_b200.synthetic import sets_workload, materialize_sets
        rng = np.random.default_rng(seed)
        pool = [rng.integers(0, 256, size=32, dtype=np.uint8).tobytes() for _ in range(k)]
        work = sets_workload(key_counts, V, seed=seed)
        work["msgs"] = b"".join(pool[g] for g in assign)
        ab = materialize_sets(work, self.table96, self.bls.sign)
        rands = rng.integers(1, 2 ** 64 - 1, size=len(assign), dtype=np.uint64, endpoint=True)
        return ab, pool, np.asarray(assign), rands

    def oracle_gt(self, sigs, msgs, pks, offs, rands):
        t0 = time.perf_counter()
        ok, gt = O.bls_verify_signature_sets(sigs, msgs, pks, offs, rands, want_gt=True)
        self.oracle_sets += len(offs) - 1
        print(f"oracle: {len(offs) - 1} sets in {time.perf_counter() - t0:.1f} s")
        return ok, gt

    def oracle_status(self, sigs, msgs, pks, offs, rands):
        ok, st = O.bls_verify_signature_sets(sigs, msgs, pks, offs, rands, want_status=True)
        self.oracle_sets += len(offs) - 1
        return ok, st


@pytest.fixture(scope="module")
def ctx(gpu):
    from lighthouse_b200 import bls
    c = Ctx(bls)
    t0 = time.perf_counter()
    yield c
    print(f"\n{__name__}: {time.perf_counter() - t0:.0f} s, {c.oracle_sets} oracle sets")
    c.table.destroy()


def ragged_counts(rng, n):
    kc = rng.integers(1, 4, size=n)
    kc[rng.choice(n, size=min(n, 1 + n // 2000), replace=False)] = 128
    kc[rng.choice(n, size=min(n, 1 + n // 8000), replace=False)] = 512
    return kc


def third_in_one(rng, m):
    """3m sets over m messages: message 0 takes a third of the sets, every other message at least one"""
    n = 3 * m
    perm = rng.permutation(n)
    assign = np.zeros(n, dtype=np.int64)
    if m > 1:
        rest = perm[m:]
        assign[rest[:m - 1]] = np.arange(1, m)
        assign[rest[m - 1:]] = rng.integers(1, m, size=len(rest) - (m - 1))
    return assign


def contributing_msgs(pool, assign):
    """set i verified against the next pool message (one message: its first bit flipped)"""
    k = len(pool)
    if k == 1:
        return flip(pool[0]) * len(assign)
    return b"".join(pool[(g + 1) % k] for g in assign)


def group_ends(assign):
    """first and last member of every group"""
    pos = set()
    for g in np.unique(assign):
        idx = np.nonzero(assign == g)[0]
        pos |= {int(idx[0]), int(idx[-1])}
    return sorted(pos)


def with_edge_rands(rands, positions):
    r = rands.copy()
    for k, i in enumerate(positions):
        r[i] = EDGE_RANDS[k % len(EDGE_RANDS)]
    return r


def grouped_case(ctx, ab, pool, assign, rands, indexed=True, want=None):
    """valid batch -> GT one; every-group-contributes batch -> the oracle's GT (explicit keys, and the pubkey table)"""
    bls = ctx.bls
    n, K = len(assign), int(ab.offsets[-1])
    ok, st, gt, plan = run_batch(bls, n, K, lambda b: b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, rands))
    assert ok is True and not st.any() and gt == GT_ONE, n
    if want:
        check_plan(plan, want, f"n = {n}, {len(pool)} messages")
    msgs = contributing_msgs(pool, assign)
    o_ok, o_gt = ctx.oracle_gt(ab.sigs, msgs, ab.pks, ab.offsets, rands)
    assert not o_ok and o_gt != GT_ONE
    ok, st, gt, p = run_batch(bls, n, K, lambda b: b.upload(ab.sigs, msgs, ab.pks, ab.offsets, rands))
    assert p["groups"] == len(pool)
    assert ok is False and not st.any() and gt == o_gt, f"n = {n}, {len(pool)} messages: GT differs from the oracle"
    if indexed:
        idx = ab.committees.reshape(-1)
        ok, st, gt, p = run_batch(bls, n, K,
                                  lambda b: b.upload_indexed(ctx.table, ab.sigs, msgs, idx, ab.offsets, rands))
        assert p["key"] == "k_pk_aggregate_indexed" and p["groups"] == len(pool)
        assert ok is False and not st.any() and gt == o_gt, f"n = {n}: indexed keys, GT differs"
    return plan, msgs, o_gt


@pytest.mark.parametrize("label", [s[0] for s in GROUP_SEAMS])
def test_group_seam_gt_parity(ctx, label):
    m = dict(GROUP_SEAMS)[label](ctx.n_sm)
    n = 3 * m
    rng = np.random.default_rng(0x6E0 + m)
    assign = third_in_one(rng, m)
    ab, pool, assign, rands = ctx.batch(ragged_counts(rng, n), assign, m, seed=0x6E0 + m)
    rands = with_edge_rands(rands, group_ends(assign)[:3 * 64])
    want = want_plan(n, m, ctx.n_sm)
    want["group_sum_levels"] = tree_levels(int(np.bincount(assign).max()))
    grouped_case(ctx, ab, pool, assign, rands, want=want)


def test_one_group_of_100k_sets(ctx):
    """100 000 single-key sets over one message: a six-level group-sum tree, one hash and one Miller loop"""
    n = 100_000
    ab, pool, assign, rands = ctx.batch(np.ones(n, dtype=np.int64), np.zeros(n, dtype=np.int64), 1, seed=0x6E1)
    plan, _, _ = grouped_case(ctx, ab, pool, assign, rands, indexed=False,
                              want=dict(groups=1, hash="k_hash_to_g2_warp", miller="k_miller_warp",
                                        key="k_pk_aggregate", sig="k_sig_prepare"))
    assert plan["group_sum_levels"] >= 2, plan


def test_100k_sets_x_128_keys_over_2048_messages(ctx):
    """an epoch's distinct AttestationData: 100 000 aggregates of 128 keys over 2 048 messages"""
    n, m = 100_000, 2048
    rng = np.random.default_rng(0x6E2)
    assign = rng.integers(0, m, size=n)
    assign[rng.permutation(n)[:m]] = np.arange(m)
    ab, pool, assign, rands = ctx.batch(np.full(n, 128), assign, m, seed=0x6E2)
    grouped_case(ctx, ab, pool, assign, rands, indexed=False, want=want_plan(n, m, ctx.n_sm))


def build_sets(ctx, sets):
    """explicit sets [(key indices into table_ext, message)] -> (sigs, msgs, pks, offsets, indices)"""
    sks = [B.interop_secret_key(i) for i in range(V)] + [(B.R - B.interop_secret_key(0)) % B.R]
    agg = [sum(sks[i] for i in keys) % B.R for keys, _ in sets]
    msgs = b"".join(m for _, m in sets)
    sigs = ctx.bls.sign(b"".join(a.to_bytes(32, "big") for a in agg), msgs)
    idx = np.array([i for keys, _ in sets for i in keys], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum([len(k) for k, _ in sets])]).astype(np.uint32)
    return sigs, msgs, ctx.table_ext[idx].tobytes(), offs, idx


def test_edge_groups_match_oracle(ctx):
    """a group whose sum is O ((pk_0) and (-pk_0) with equal scalars), a group of two identical sets (the doubling
    branch), a group where those meet a third set, and scalars 1, 2^63, 2^64-1 on the first and last members.
    Equal r_i apk_i come with equal r_i sig_i, and the warp-mode sum of r_i sig_i (k_g2_sum_warp, up to 6 x SMs sets)
    takes distinct points for granted (the scalars are secret and random), so the batch is sized for k_g2_reduce."""
    rng = np.random.default_rng(0x6E3)
    n_msgs = 12 + 120
    pool = [rng.integers(0, 256, size=32, dtype=np.uint8).tobytes() for _ in range(n_msgs)]
    sets = [([0], pool[0]), ([V], pool[0]),                     # sum O
            ([5], pool[1]), ([5], pool[1]),                     # P + P
            ([0], pool[2]), ([V], pool[2]), ([9, 10], pool[2])]  # O + Q
    for g in range(3, n_msgs):
        for _ in range(int(rng.integers(1, 6)) if g < 12 else 8):
            sets.append((sorted(rng.choice(V, size=int(rng.integers(1, 4)), replace=False).tolist()), pool[g]))
    n = len(sets)
    assert n > 6 * ctx.n_sm
    sigs, msgs, pks, offs, idx = build_sets(ctx, sets)
    assign = np.array([pool.index(m) for _, m in sets])
    rands = rng.integers(1, 2 ** 64 - 1, size=n, dtype=np.uint64, endpoint=True)
    rands[1] = rands[0]; rands[5] = rands[4]; rands[3] = rands[2]
    rands = with_edge_rands(rands, [i for i in group_ends(assign) if i > 6])
    r_max = rands.copy()
    r_max[7:] = np.uint64(EDGE_RANDS[2])                         # every other member at 2^64 - 1
    for r in (rands, r_max):
        ok, st, gt, plan = run_batch(ctx.bls, n, len(idx), lambda b: b.upload(sigs, msgs, pks, offs, r))
        assert plan["sum"] == "k_g2_reduce" and plan["groups"] == n_msgs, plan
        assert ok is True and not st.any() and gt == GT_ONE
        vmsgs = contributing_msgs(pool, assign)
        _, o_gt = ctx.oracle_gt(sigs, vmsgs, pks, offs, r)
        for up in (lambda b: b.upload(sigs, vmsgs, pks, offs, r),
                   lambda b: b.upload_indexed(ctx.table, sigs, vmsgs, idx, offs, r)):
            ok, st, gt, plan = run_batch(ctx.bls, n, len(idx), up)
            assert ok is False and not st.any() and gt == o_gt and plan["groups"] == n_msgs


# ---- per-set statuses inside groups -------------------------------------------------------------------------------
def status_mix(ctx, n, k, big):
    """every status code and the pairs 1+4, 2+6, 3+5, 1+6, once on a member next to passing members and once on every
    member of a group -> (sigs, msgs, offsets, indices into table_ext (V + 1 = past the end), pks, rands, assign)"""
    rng = np.random.default_rng(0x6E4 + n)
    kc = ragged_counts(rng, n)
    if big:                                                   # >= 2^20 keys: at least 3 chunks of the streamed upload
        kc[:] = 512
    assign = rng.integers(0, k, size=n)
    assign[rng.permutation(n)[:k]] = np.arange(k)
    ab, pool, assign, rands = ctx.batch(kc, assign, k, seed=0x6E4 + n)
    offs = ab.offsets
    sets_idx = [list(ab.committees.reshape(-1)[offs[i]:offs[i + 1]]) for i in range(n)]
    sigs = bytearray(ab.sigs)
    bad_g2 = B.g2_compress(_non_subgroup_g2())
    groups = [np.nonzero(assign == g)[0] for g in range(k)]
    multi = [g for g in groups if len(g) >= 3]
    assert len(multi) >= 2 * len(MIX)
    targets = [[int(g[len(g) // 2])] for g in multi[:len(MIX)]] + [list(map(int, g)) for g in multi[len(MIX):2 * len(MIX)]]
    for t, members in enumerate(targets):
        sc, kcode = MIX[t % len(MIX)]
        for i in members:
            s = ab.sigs[96 * i:96 * i + 96]
            if sc:
                sigs[96 * i:96 * i + 96] = {1: bytes(96), 2: bytes([s[0] & 0x7F]) + s[1:], 3: bad_g2}[sc]
            if kcode == 4:
                sets_idx[i] = []
            elif kcode == 5:
                sets_idx[i] = [0, V]                          # pk_0 + (-pk_0)
            elif kcode == 6:
                sets_idx[i] = [sets_idx[i][0], V + 1]         # past the table / compression flag set
    idx = np.array([j for s in sets_idx for j in s], dtype=np.uint32)
    new_offs = np.concatenate([[0], np.cumsum([len(s) for s in sets_idx])]).astype(np.uint32)
    bad_key = ctx.table_ext[1].copy()
    bad_key[0] |= 0x80
    pks = np.vstack([ctx.table_ext, bad_key[None]])[idx]
    return bytes(sigs), ab.msgs, new_offs, idx, pks.tobytes(), rands, assign


@pytest.mark.parametrize("n,k,big", [(300, 40, False), (2200, 200, True)])
def test_status_mix_in_groups_matches_oracle(ctx, n, k, big):
    sigs, msgs, offs, idx, pks, rands, assign = status_mix(ctx, n, k, big)
    o_ok, o_st = ctx.oracle_status(sigs, msgs, pks, offs, rands)
    assert not o_ok and sorted(set(o_st) - {0}) == [1, 2, 3, 4, 5, 6]
    K = len(idx)
    runs = {
        "explicit": lambda b: b.upload(sigs, msgs, pks, offs, rands),
        "indexed": lambda b: b.upload_indexed(ctx.table, sigs, msgs, idx, offs, rands),
        "streamed": lambda b: b.upload_async(sigs, msgs, pks, offs, rands),
    }
    for name, up in runs.items():
        ok, st, _, plan = run_batch(ctx.bls, n, K, up)
        assert plan["groups"] == k, (name, plan)
        if big and name == "streamed":
            assert plan["key_chunks"] >= 3, plan
        assert ok is False, name
        np.testing.assert_array_equal(st, o_st, err_msg=f"{name} ({plan['key']}, n = {n})")
    ok, st = ctx.bls.verify_signature_sets_raw(sigs, msgs, pks, offs, rands, want_status=True)
    assert ok is False
    np.testing.assert_array_equal(st, o_st, err_msg="lhb200_verify_signature_sets")


def test_plugin_call_and_resident_inputs(ctx):
    """10 000 sets over 40 messages (hash and Miller in latency mode, signatures and keys per set): the one-shot
    lhb200_verify_signature_sets gives the oracle's verdicts, and inputs bound with set_device_inputs are not grouped
    but give the same GT"""
    import torch
    n, k = 10_000, 40
    rng = np.random.default_rng(0x6E5)
    assign = rng.integers(0, k, size=n)
    assign[rng.permutation(n)[:k]] = np.arange(k)
    ab, pool, assign, rands = ctx.batch(ragged_counts(rng, n), assign, k, seed=0x6E5)
    want = want_plan(n, k, ctx.n_sm)
    assert want["hash"] == "k_hash_to_g2_warp" and want["miller"] == "k_miller_warp"
    _, msgs, o_gt = grouped_case(ctx, ab, pool, assign, rands, indexed=False, want=want)
    assert ctx.bls.verify_signature_sets_raw(ab.sigs, ab.msgs, ab.pks, ab.offsets, rands) is True
    assert ctx.bls.verify_signature_sets_raw(ab.sigs, msgs, ab.pks, ab.offsets, rands) is False
    dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    d = [dev(ab.sigs), dev(msgs), dev(ab.pks), dev(np.asarray(ab.offsets, dtype=np.uint32).tobytes()),
         dev(rands.tobytes())]
    torch.cuda.synchronize()
    ok, st, gt, plan = run_batch(ctx.bls, n, int(ab.offsets[-1]),
                                 lambda b: b.set_device_inputs(*[t.data_ptr() for t in d], n))
    assert plan["groups"] == 0 and plan["group_sum"] == "" and plan["hash"] == want_plan(n, n, ctx.n_sm)["hash"]
    assert ok is False and not st.any() and gt == o_gt


def test_switch_off_gives_identical_outputs(ctx, tmp_path):
    """LHB_GROUP_MESSAGES=0 (scripts/regime_probe.py in a subprocess): no grouping, the same GT and statuses"""
    m = 256
    rng = np.random.default_rng(0x6E6)
    assign = third_in_one(rng, m)
    ab, pool, assign, rands = ctx.batch(ragged_counts(rng, 3 * m), assign, m, seed=0x6E6)
    _, msgs, o_gt = grouped_case(ctx, ab, pool, assign, rands, indexed=False)
    cases = {}
    f = tmp_path / "gt.npz"
    np.savez(f, sigs=np.frombuffer(ab.sigs, np.uint8), msgs=np.frombuffer(msgs, np.uint8),
             pks=np.frombuffer(ab.pks, np.uint8), offsets=ab.offsets, rands=rands)
    cases[f.name] = ("gt", o_gt.hex())
    sigs, smsgs, offs, idx, pks, srands, _ = status_mix(ctx, 300, 40, False)
    _, o_st = ctx.oracle_status(sigs, smsgs, pks, offs, srands)
    f = tmp_path / "mix.npz"
    np.savez(f, sigs=np.frombuffer(sigs, np.uint8), msgs=np.frombuffer(smsgs, np.uint8),
             pks=np.frombuffer(pks, np.uint8), offsets=offs, rands=srands)
    cases[f.name] = ("status", bytes(o_st).hex())
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "regime_probe.py")] +
                         [str(tmp_path / name) for name in cases],
                         env=dict(os.environ, LHB_GROUP_MESSAGES="0"), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]
    assert [r["file"] for r in rows] == list(cases)
    for r in rows:
        kind, ref = cases[r["file"]]
        assert r["plan"]["groups"] == 0 and r["plan"]["group_sum"] == "" and r["ok"] is False, r["file"]
        if kind == "gt":
            assert r["status"] == "00" * r["n"] and r["gt"] == ref
        else:
            assert r["status"] == ref
