"""GPU: the batch verifier at both sides of every seam where lhb200_bls_batch_verify_enqueue switches kernels, compared
byte for byte with the C oracle (oracle/bls12_381.c).

The verdict alone is a weak check: a kernel that drops a set, or gives set i the scalar of set i + 1 on both sides of
the pairing equation, still accepts a valid batch and still rejects one with a single bad set.  So every size also runs
an "every set contributes" batch: set i carries the message of set i + 1, every pair is non-trivial, and the GT value
(final-exponentiated product, lhb200_bls_batch_gt) must equal the oracle's.  The sizes come from the device's SM count;
lhb200_bls_batch_plan reports which kernels ran, so each case asserts the path it exercised instead of assuming it.
"""
import functools
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import oracle_lib as O
from oracle import bls_ref as B

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = 1024                                           # validators (>= the 512-key sets)
GT_ONE = (1).to_bytes(48, "big") + bytes(576 - 48)
INF_SIG = bytes([0xC0]) + bytes(95)
EDGE_RANDS = (1, 2 ** 63, 2 ** 64 - 1)

# (label, size from the SM count, plan fields that size must produce under the default switches)
SEAMS = [
    ("one_set", lambda s: 1, dict(sig="k_sig_prepare_warp", sum="", hash="k_hash_to_g2_warp",
                                  key="k_pk_partial+k_pk_combine", miller="k_miller_warp", miller_wpb=4,
                                  final="k_final_warp", lane_sets_per_thread=1)),
    ("sum_warp_1_level", lambda s: 2, dict(sum="k_g2_sum_warp", sum_levels=1)),
    ("sum_warp_1_level_full", lambda s: 4, dict(sum="k_g2_sum_warp", sum_levels=1)),
    ("sum_warp_2_levels", lambda s: 5, dict(sum="k_g2_sum_warp", sum_levels=2)),
    ("sum_warp_2_levels_full", lambda s: 16, dict(sum="k_g2_sum_warp", sum_levels=2)),
    ("sum_warp_3_levels", lambda s: 17, dict(sum="k_g2_sum_warp", sum_levels=3)),
    ("miller_warp_4wpb_last", lambda s: 255, dict(miller="k_miller_warp", miller_wpb=4, fp12_reduce_levels=0)),
    ("miller_warp_8wpb_first", lambda s: 256, dict(miller="k_miller_warp", miller_wpb=8, fp12_reduce_levels=0)),
    ("miller_warp_no_reduce_last", lambda s: 511, dict(miller="k_miller_warp", fp12_reduce_levels=0, n_tail=64)),
    ("miller_warp_reduce_first", lambda s: 512, dict(miller="k_miller_warp", fp12_reduce_levels=1)),
    ("g2_warp_last", lambda s: 6 * s, dict(sig="k_sig_prepare_warp", hash="k_hash_to_g2_warp", sum="k_g2_sum_warp")),
    ("g2_lane_first", lambda s: 6 * s + 1, dict(sig="k_sig_prepare", hash="k_hash_to_g2_pair", sum="k_g2_reduce",
                                                miller="k_miller_warp")),
    ("miller_warp_last", lambda s: 8 * s - 1, dict(miller="k_miller_warp", miller_wpb=8)),
    ("miller_coop_first", lambda s: 8 * s, dict(miller="k_miller_coop", miller_few_warps=1, miller_rounds_cap=1,
                                                final="k_final_warp")),
    ("hash_pair_last", lambda s: 4096, dict(hash="k_hash_to_g2_pair")),
    ("hash_lane_first", lambda s: 4097, dict(hash="k_hash_to_g2")),
    ("coop_few_warps_last", lambda s: 7679, dict(miller="k_miller_coop", miller_few_warps=1)),
    ("coop_full_first", lambda s: 7680, dict(miller="k_miller_coop", miller_few_warps=0, miller_rounds_cap=1)),
    ("pk_split_last", lambda s: 8192, dict(key="k_pk_partial+k_pk_combine")),
    ("pk_lane_first", lambda s: 8193, dict(key="k_pk_aggregate")),
    ("spin_wait_last", lambda s: 16383, dict(key="k_pk_aggregate")),
    ("blocking_wait_first", lambda s: 16384, dict(key="k_pk_aggregate")),
    ("coop_one_round_last", lambda s: 240 * s - 1, dict(miller="k_miller_coop", miller_rounds_cap=1)),
    ("coop_two_rounds_first", lambda s: 240 * s, dict(miller="k_miller_coop", miller_rounds_cap=2)),
    ("cta_cap_first", lambda s: 768 * s + 1, dict(lane_sets_per_thread=2, sig="k_sig_prepare", hash="k_hash_to_g2",
                                                  key="k_pk_aggregate")),
]
SEAM = {label: (size, want) for label, size, want in SEAMS}
# every kernel the default switches can choose (the TMA key kernel, k_miller_multi and k_final_coop are opt-in: they
# run in test_switch_variants_match_oracle)
DEFAULT_KERNELS = {
    "sig": {"k_sig_prepare", "k_sig_prepare_warp"}, "sum": {"k_g2_reduce", "k_g2_sum_warp"},
    "hash": {"k_hash_to_g2", "k_hash_to_g2_pair", "k_hash_to_g2_warp"},
    "key": {"k_pk_aggregate", "k_pk_partial+k_pk_combine", "k_pk_aggregate_indexed"},
    "miller": {"k_miller_warp", "k_miller_coop"}, "final": {"k_final_warp"},
}


class Ctx:
    """Inputs, oracle values and plans shared by the tests of this module (built on first use)."""

    def __init__(self, bls):
        from lighthouse_b200.synthetic import interop_pubkey_table
        self.bls = bls
        self.table96 = interop_pubkey_table(V)
        neg0 = self.table96[0].copy()                          # -pk_0: a key list (pk_0, -pk_0) sums to infinity
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
        self.plans = {}
        self.oracle_sets = 0
        O.set_threads(O.hw_threads())

    @functools.lru_cache(maxsize=None)
    def inputs(self, n, big=False):
        """n ragged sets, mostly 1-3 keys with a few of 128 and 512; big=True: enough 512-key sets for >= 3 chunks
        of the streamed upload (1 048 576 keys)."""
        from lighthouse_b200.synthetic import sets_workload, materialize_sets
        rng = np.random.default_rng(0x5EA0 + n + (1 << 20) * big)
        kc = rng.integers(1, 4, size=n)
        kc[rng.choice(n, size=min(n, 1 + n // 2000), replace=False)] = 128
        kc[rng.choice(n, size=min(n, 2100 if big else 1 + n // 8000), replace=False)] = 512
        work = sets_workload(kc, V, seed=0x5EA0 + n)
        ab = materialize_sets(work, self.table96, self.bls.sign)
        rands = rng.integers(1, 2 ** 64 - 1, size=n, dtype=np.uint64, endpoint=True)
        return ab, rands

    def oracle_gt(self, sigs, msgs, pks, offs, rands):
        t0 = time.perf_counter()
        ok, gt = O.bls_verify_signature_sets(sigs, msgs, pks, offs, rands, want_gt=True)
        self.oracle_sets += len(offs) - 1
        print(f"oracle: {len(offs) - 1} sets in {time.perf_counter() - t0:.1f} s ({O.hw_threads()} threads)")
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


def rotated(msgs, n):
    """set i gets the message of set i + 1 (mod n); a single set gets its message with one bit flipped"""
    if n == 1:
        return bytes([msgs[0] ^ 1]) + msgs[1:]
    return msgs[32:] + msgs[:32]


def boundary_sets(n, plan):
    """first and last set, and the sets on each side of the block / warp / chunk boundaries the plan reports"""
    steps = {4, 8, 64, plan["lane_grid"] * 64}
    if plan["miller"] == "k_miller_warp":
        steps |= {plan["miller_wpb"], plan["miller_wpb"] * plan["miller_grid"]}
    elif plan["miller"] == "k_miller_coop":
        steps |= {plan["miller_spw"], plan["miller_spw"] * plan["miller_grid"]}
    pos = {0, n - 1}
    for st in steps:
        for b in (st, 2 * st, 3 * st, (n - 1) // st * st):
            if 0 < b < n:
                pos |= {b - 1, b}
    return sorted(pos)


def with_edge_rands(rands, positions):
    r = rands.copy()
    for k, i in enumerate(positions):
        r[i] = EDGE_RANDS[k % len(EDGE_RANDS)]
    return r


def run_batch(bls, n, n_keys, upload):
    b = bls.Batch(n, max(n_keys, 1))        # sized exactly: a read past the batch meets unwritten memory
    try:
        upload(b)
        b.enqueue()
        ok, st = b.result(want_status=True)
        return ok, st.copy(), (b.gt_bytes() if not st.any() else None), b.plan()
    finally:
        b.destroy()


def check_plan(plan, want, what):
    got = {k: plan[k] for k in want}
    assert got == want, f"{what}: plan {plan} does not match {want}"


def seam_case(ctx, label):
    """valid batch (GT one) and every-set-contributes batch (GT == oracle), explicit keys, then the same through the
    pubkey table -> (n, plan, rands, oracle GT of the rotated batch)"""
    bls = ctx.bls
    size, want = SEAM[label]
    n = size(ctx.n_sm)
    ab, rands = ctx.inputs(n)
    K = int(ab.offsets[-1])
    ok, st, gt, plan = run_batch(bls, n, K, lambda b: b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, rands))
    assert ok is True and not st.any() and gt == GT_ONE, (label, n)
    assert plan["n_sets"] == n
    check_plan(plan, want, f"{label} (n = {n})")
    ctx.plans[label] = plan
    r = with_edge_rands(rands, boundary_sets(n, plan))
    ok, st, gt, _ = run_batch(bls, n, K, lambda b: b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, r))
    assert ok is True and not st.any() and gt == GT_ONE, (label, n, "edge scalars")
    msgs = rotated(ab.msgs, n)
    o_ok, o_gt = ctx.oracle_gt(ab.sigs, msgs, ab.pks, ab.offsets, r)
    assert not o_ok and o_gt != GT_ONE
    ok, st, gt, _ = run_batch(bls, n, K, lambda b: b.upload(ab.sigs, msgs, ab.pks, ab.offsets, r))
    assert ok is False and not st.any(), (label, n)
    assert gt == o_gt, f"{label} (n = {n}): GT differs from the oracle"
    idx = ab.committees.reshape(-1)
    ok, st, gt, p = run_batch(bls, n, K, lambda b: b.upload_indexed(ctx.table, ab.sigs, msgs, idx, ab.offsets, r))
    assert p["key"] == "k_pk_aggregate_indexed"
    assert ok is False and not st.any() and gt == o_gt, f"{label} (n = {n}): indexed keys, GT differs"
    return n, plan, r, o_gt


@pytest.mark.parametrize("label", [s[0] for s in SEAMS])
def test_seam_gt_parity(ctx, label):
    seam_case(ctx, label)


def test_default_plans_cover_every_variant(ctx):
    """over the sweep, every kernel the default switches can choose ran, and both sides of every shape switch"""
    plans = {}
    for label, size, _ in SEAMS:
        if label not in ctx.plans:                          # module run with -k: take the plan of the valid batch
            n = size(ctx.n_sm)
            ab, rands = ctx.inputs(n)
            ctx.plans[label] = run_batch(ctx.bls, n, int(ab.offsets[-1]),
                                         lambda b: b.upload(ab.sigs, ab.msgs, ab.pks, ab.offsets, rands))[3]
        plans[label] = ctx.plans[label]
    seen = {f: {p[f] for p in plans.values()} for f in DEFAULT_KERNELS}
    seen["key"].add("k_pk_aggregate_indexed")               # every seam case also runs the pubkey-table path
    for f, kernels in DEFAULT_KERNELS.items():
        assert kernels <= seen[f], f"{f}: {kernels - seen[f]} never ran"
    for f, values in (("miller_wpb", {4, 8}), ("miller_few_warps", {0, 1}), ("miller_rounds_cap", {1, 2}),
                      ("lane_sets_per_thread", {1, 2})):
        assert values <= {p[f] for p in plans.values()}, f
    assert {p["fp12_reduce_levels"] > 0 for p in plans.values()} == {False, True}


@pytest.mark.parametrize("label", ["sum_warp_3_levels", "miller_coop_first", "hash_lane_first"])
def test_all_infinity_signatures(ctx, label):
    """every signature is the infinity encoding: the sum tree is all infinity, the pair (-g1, sum r sig) drops out, and
    the GT value is still the oracle's"""
    size, _ = SEAM[label]
    n = size(ctx.n_sm)
    ab, rands = ctx.inputs(n)
    sigs = INF_SIG * n
    o_ok, o_gt = ctx.oracle_gt(sigs, ab.msgs, ab.pks, ab.offsets, rands)
    ok, st, gt, _ = run_batch(ctx.bls, n, int(ab.offsets[-1]),
                              lambda b: b.upload(sigs, ab.msgs, ab.pks, ab.offsets, rands))
    assert ok is False and not o_ok and not st.any()
    assert gt == o_gt


@pytest.mark.parametrize("n", [2200, 8193])
def test_streamed_upload_chunks_match_oracle(ctx, n):
    """lhb200_bls_batch_upload_async with >= 3 key chunks (more than 2^20 keys, ragged counts), on both key kernels:
    the GT equals the blocking upload's and the oracle's"""
    ab, rands = ctx.inputs(n, big=True)
    K = int(ab.offsets[-1])
    assert K >= 1 << 20
    msgs = rotated(ab.msgs, n)
    o_ok, o_gt = ctx.oracle_gt(ab.sigs, msgs, ab.pks, ab.offsets, rands)
    ok, st, gt, plan = run_batch(ctx.bls, n, K, lambda b: b.upload_async(ab.sigs, msgs, ab.pks, ab.offsets, rands))
    assert plan["key_chunks"] >= 3, plan
    assert plan["key"] == ("k_pk_partial+k_pk_combine" if n <= 8192 else "k_pk_aggregate"), plan
    assert ok is False and not st.any() and gt == o_gt
    ok, st, gt, plan = run_batch(ctx.bls, n, K, lambda b: b.upload(ab.sigs, msgs, ab.pks, ab.offsets, rands))
    assert plan["key_chunks"] == 0 and gt == o_gt


# ---- per-set statuses ---------------------------------------------------------------------------------------------
# single codes and the pairs where the signature and the key stage both fail: the signature's code must win, whatever
# order the two concurrent stages finish in (no rerun loops: the fix is that they write separate arrays)
MIX = [(1, 0), (2, 0), (3, 0), (0, 4), (0, 5), (0, 6), (1, 4), (2, 6), (3, 5), (1, 6)]


def _non_subgroup_g2():
    x = (3, 1)
    while True:
        y = B.f2_sqrt(B.f2_add(B.f2_mul(B.f2_sqr(x), x), B.B2))
        if y:
            return (x, y)
        x = (x[0] + 1, 1)


def status_mix(ctx, n):
    """-> (sigs, msgs, offsets, indices into ctx.table_ext (V + 1 = past the end), explicit pks, rands, positions)"""
    ab, rands = ctx.inputs(n)
    offs = ab.offsets
    sets_idx = [list(ab.committees.reshape(-1)[offs[i]:offs[i + 1]]) for i in range(n)]
    sigs = bytearray(ab.sigs)
    bad_g2 = B.g2_compress(_non_subgroup_g2())
    pos = sorted({0, 1, 3, 4, 5, 63, 64, 65, 127, 128, 255, 256, n // 2, n - 3, n - 2, n - 1} & set(range(n)))
    for k, i in enumerate(pos):
        sc, kc = MIX[k % len(MIX)]
        s = ab.sigs[96 * i:96 * i + 96]
        if sc:
            sigs[96 * i:96 * i + 96] = {1: bytes(96), 2: bytes([s[0] & 0x7F]) + s[1:], 3: bad_g2}[sc]
        if kc == 4:
            sets_idx[i] = []
        elif kc == 5:
            sets_idx[i] = [0, V]                             # pk_0 + (-pk_0)
        elif kc == 6:
            sets_idx[i] = [sets_idx[i][0], V + 1]            # second key: past the table / compression flag set
    idx = np.array([j for s in sets_idx for j in s], dtype=np.uint32)
    new_offs = np.concatenate([[0], np.cumsum([len(s) for s in sets_idx])]).astype(np.uint32)
    bad_key = ctx.table_ext[1].copy()
    bad_key[0] |= 0x80                                       # compression flag on an uncompressed key
    pks = np.vstack([ctx.table_ext, bad_key[None]])[idx]
    return bytes(sigs), ab.msgs, new_offs, idx, pks.tobytes(), rands, pos


@pytest.mark.parametrize("n", [300, 8193])
def test_status_precedence_matches_oracle(ctx, n):
    """each status code and the pairs 1+4, 2+6, 3+5, 1+6 at seam positions, through the split / per-set key kernels,
    the pubkey table and the streamed upload: the device statuses equal the oracle's"""
    sigs, msgs, offs, idx, pks, rands, pos = status_mix(ctx, n)
    o_ok, o_st = ctx.oracle_status(sigs, msgs, pks, offs, rands)
    assert not o_ok and sorted(set(o_st[pos])) == [1, 2, 3, 4, 5, 6]
    K = len(idx)
    runs = {
        "explicit": lambda b: b.upload(sigs, msgs, pks, offs, rands),
        "indexed": lambda b: b.upload_indexed(ctx.table, sigs, msgs, idx, offs, rands),
        "streamed": lambda b: b.upload_async(sigs, msgs, pks, offs, rands),
    }
    for name, up in runs.items():
        ok, st, _, plan = run_batch(ctx.bls, n, K, up)
        assert ok is False, name
        np.testing.assert_array_equal(st, o_st, err_msg=f"{name} ({plan['key']}, n = {n})")


# ---- the other kernel families, one subprocess per switch set -------------------------------------------------------
VARIANTS = [
    ({"LHB_MILLER_WARP": "0"}, dict(miller="k_miller_coop")),
    ({"LHB_G2_WARP": "0"}, dict(sig="k_sig_prepare", hash="k_hash_to_g2_pair")),
    ({"LHB_FINAL_WARP": "0"}, dict(final="k_final_coop")),
    ({"LHB_PK_TMA": "1"}, dict(key="k_pk_aggregate_tma")),
    ({"LHB_MILLER_COOP": "0"}, dict(miller="k_miller_multi", last_miller=1, final="k_final_coop")),
]
VARIANT_SEAMS = ["one_set", "sum_warp_3_levels", "miller_warp_8wpb_first", "g2_lane_first", "miller_coop_first"]


def test_switch_variants_match_oracle(ctx, tmp_path):
    """scripts/regime_probe.py under each switch set: the plan shows the variant ran, the GT of every-set-contributes
    batches equals the oracle's, and the status mix gives the oracle's statuses"""
    cases = {}
    for label in VARIANT_SEAMS:
        size, _ = SEAM[label]
        n = size(ctx.n_sm)
        ab, rands = ctx.inputs(n)
        msgs = rotated(ab.msgs, n)
        _, o_gt = ctx.oracle_gt(ab.sigs, msgs, ab.pks, ab.offsets, rands)
        f = tmp_path / f"{label}.npz"
        np.savez(f, sigs=np.frombuffer(ab.sigs, np.uint8), msgs=np.frombuffer(msgs, np.uint8),
                 pks=np.frombuffer(ab.pks, np.uint8), offsets=ab.offsets, rands=rands)
        cases[f.name] = ("gt", o_gt.hex())
    sigs, msgs, offs, idx, pks, rands, _ = status_mix(ctx, 300)
    _, o_st = ctx.oracle_status(sigs, msgs, pks, offs, rands)
    f = tmp_path / "mix.npz"
    np.savez(f, sigs=np.frombuffer(sigs, np.uint8), msgs=np.frombuffer(msgs, np.uint8), pks=np.frombuffer(pks, np.uint8),
             offsets=offs, rands=rands)
    cases[f.name] = ("status", bytes(o_st).hex())
    files = [str(tmp_path / name) for name in cases]
    for env, want in VARIANTS:
        out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "regime_probe.py")] + files,
                             env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, (env, out.stderr[-2000:])
        rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]
        assert [r["file"] for r in rows] == list(cases), env
        for r in rows:
            kind, ref = cases[r["file"]]
            check_plan(r["plan"], want, f"{env} {r['file']}")
            assert r["ok"] is False, (env, r["file"])
            if kind == "gt":
                assert r["status"] == "00" * r["n"] and r["gt"] == ref, f"{env} {r['file']}: GT differs"
            else:
                assert r["status"] == ref, f"{env}: statuses {r['status']} != oracle {ref}"
