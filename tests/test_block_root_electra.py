"""BeaconBlockElectra / BlindedBeaconBlockElectra canonical_root (beacon_block_body.rs:70-121, attestation.rs:76-82,
execution_payload.rs:54-101): the Electra arm of the fork-parametrised block describer and the DepositRequest record
kind, checked against the generic from-spec merkleization of tests/ssz_spec.py over the decoded value."""
import pytest

from lighthouse_b200 import ssz_schema as S
from lighthouse_b200 import synthetic
from tests import ssz_spec

T, BT = S.BEACON_BLOCK_BY_FORK["electra"], S.BEACON_BLOCK_BODY_BY_FORK["electra"]
BLINDED_T = S.BLINDED_BEACON_BLOCK_BY_FORK["electra"]
PT = dict(S.ExecutionPayloadElectra[1])
NO_DENEB_OPS = dict(n_transactions=0, n_proposer_slashings=0, n_deposits=0, n_exits=0, n_bls_changes=0, n_withdrawals=0,
                    n_blobs=0, extra_data_len=0)
SHAPES = {
    # 8 attestations over 6 committees each, 1 attester slashing, 16 withdrawal requests, 1 consolidation
    "mainnet_like": dict(seed=51, committees_per_attestation=6, bits_per_committee=480, n_deposit_requests=5),
    "empty": dict(seed=52, n_attestations=0, n_attester_slashings=0, n_deposit_requests=0, n_withdrawal_requests=0,
                  n_consolidations=0, **NO_DENEB_OPS),
    # aggregation-bit lengths across byte / chunk boundaries, past the pre-Electra limit of 2048, and at 131 072
    "bit_lengths": dict(seed=53, bit_lengths=[0, 1, 255, 256, 257, 2048, 2049, 131072], n_transactions=3),
    # an attester slashing whose first indexed attestation has 131 072 indices (1 MB)
    "max_slashing": dict(seed=54, n_attestations=1, slashing_indices=131072, n_transactions=3),
}
# 64 / 65: container ops / record kernel; 256 / 257: a power of two and one past it; 8192: the limit (1.5 MB)
DEPOSIT_REQUEST_COUNTS = [0, 1, 8, 9, 64, 65, 256, 257, 8192]


def _block(**kw):
    return synthetic.beacon_block_electra(**kw)


def _want(value):
    return ssz_spec.hash_tree_root(T, value), ssz_spec.hash_tree_root(BT, value["body"])


def _blind(value):
    ep = value["body"]["execution_payload"]
    roots = [ssz_spec.hash_tree_root(PT[k], ep[k])
             for k in ("transactions", "withdrawals", "deposit_requests", "withdrawal_requests")]
    return synthetic.blind_block_electra(value, *roots)


def test_electra_block_schema_roundtrip_and_blinded_root():
    """Host side (no GPU): the generator's SSZ decodes and re-encodes under the Electra descriptors, the layouts have
    the reference's field counts and fixed parts, and the blinded block has the full block's root."""
    assert len(BT[1]) == 13 and len(S.ExecutionPayloadElectra[1]) == 19 and len(S.ExecutionPayloadHeaderElectra[1]) == 19
    assert [S.fixed_size(t) for t in (BT, S.ExecutionPayloadElectra, S.ExecutionPayloadHeaderElectra,
                                      S.AttestationElectra, S.DepositRequest, S.ExecutionLayerWithdrawalRequest,
                                      S.SignedConsolidation)] == [396, 536, 648, 236, 192, 76, 120]
    for kw in (dict(seed=41, n_transactions=5, bits_per_committee=40, n_deposit_requests=9), dict(SHAPES["empty"])):
        v, ssz = _block(**kw)
        assert S.serialize(T, ssz_spec.deserialize(T, ssz)) == ssz
        bv, bssz = _blind(v)
        assert S.serialize(BLINDED_T, ssz_spec.deserialize(BLINDED_T, bssz)) == bssz
        assert ssz_spec.hash_tree_root(BLINDED_T, bv) == ssz_spec.hash_tree_root(T, v)


def _check_single(value, ssz):
    from lighthouse_b200 import tree_hash
    want, want_body = _want(value)
    assert tree_hash.beacon_block_roots([ssz], "electra", want_body_roots=True) == ([want], [want_body])
    _, bssz = _blind(value)
    assert tree_hash.beacon_block_roots([bssz], "electra", want_body_roots=True, blinded=True) == ([want], [want_body])
    return want, want_body, bssz


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_gpu_electra_block_root(gpu, name):
    _check_single(*_block(**SHAPES[name]))


@pytest.mark.gpu
@pytest.mark.parametrize("n", DEPOSIT_REQUEST_COUNTS)
def test_gpu_electra_deposit_requests(gpu, n):
    _check_single(*_block(seed=60 + n % 97, n_deposit_requests=n, n_transactions=4, bits_per_committee=100))


@pytest.mark.gpu
def test_gpu_electra_shapes_in_one_batch(gpu):
    """Every shape above, full and blinded, as one batch each: roots, body roots and order."""
    from lighthouse_b200 import tree_hash
    kws = [SHAPES[k] for k in sorted(SHAPES)] + [dict(seed=70, n_deposit_requests=n, n_transactions=2)
                                               for n in DEPOSIT_REQUEST_COUNTS]
    values, blobs = zip(*[_block(**kw) for kw in kws])
    want, want_body = map(list, zip(*[_want(v) for v in values]))
    assert tree_hash.beacon_block_roots(blobs, "electra", want_body_roots=True) == (want, want_body)
    blinded = [_blind(v)[1] for v in values]
    assert tree_hash.beacon_block_roots(blinded, "electra", want_body_roots=True, blinded=True) == (want, want_body)


@pytest.mark.gpu
def test_gpu_full_deposit_request_list_plans_on_the_first_attempt(gpu):
    """8 192 DepositRequests (1.5 MB) fit the first arena bound of the block path: the single planning pass is not
    redone under the fallback bound (which reports itself through lhb200_last_error)."""
    from lighthouse_b200 import tree_hash, Lhb200Error
    from lighthouse_b200._ffi import lib
    value, ssz = _block(seed=71, n_deposit_requests=8192)
    with pytest.raises(Lhb200Error):
        tree_hash.beacon_block_roots([ssz[:100]], "electra")      # leaves a known message in lhb200_last_error
    before = lib.lhb200_last_error()
    assert tree_hash.beacon_block_roots([ssz, ssz], "electra") == [_want(value)[0]] * 2
    assert lib.lhb200_last_error() == before, lib.lhb200_last_error()


@pytest.mark.gpu
def test_gpu_electra_epoch_batch_and_other_fork_bytes(gpu):
    """32 Electra blocks in one pass; a Deneb block in the middle of that batch, or Electra bytes hashed as Deneb, give
    EINVAL or a different root, never the other fork's root."""
    from lighthouse_b200 import tree_hash, Lhb200Error
    from lighthouse_b200._ffi import EINVAL
    values, blobs = zip(*[_block(seed=200 + i, committees_per_attestation=1 + i % 8, n_deposit_requests=i % 11,
                                 n_transactions=20 + i) for i in range(32)])
    want = [_want(v)[0] for v in values]
    assert tree_hash.beacon_block_roots(blobs, "electra") == want
    deneb_value, deneb = synthetic.beacon_block_deneb(seed=16, n_attestations=8)
    deneb_root = ssz_spec.hash_tree_root(S.BEACON_BLOCK_BY_FORK["deneb"], deneb_value)
    mixed = list(blobs)
    mixed[16] = deneb
    try:
        got = tree_hash.beacon_block_roots(mixed, "electra")
        assert got[16] != deneb_root and got[:16] == want[:16] and got[17:] == want[17:]
    except Lhb200Error as e:
        assert e.code == EINVAL
    try:
        assert tree_hash.beacon_block_roots(blobs[:1], "deneb") != want[:1]
    except Lhb200Error as e:
        assert e.code == EINVAL


def _retyped(body=None, payload=None):
    """The Electra block descriptor with some body / payload field types replaced, to serialise over-limit values."""
    pf = [(n, (payload or {}).get(n, t)) for n, t in S.ExecutionPayloadElectra[1]]
    bf = [(n, S.C(*pf) if n == "execution_payload" else (body or {}).get(n, t)) for n, t in BT[1]]
    return S.C(*[(n, S.C(*bf)) if n == "body" else (n, t) for n, t in T[1]])


def _u32(b, at):
    return int.from_bytes(b[at:at + 4], "little")


def _malformed():
    """(label, SSZ) pairs the describer must refuse with EINVAL."""
    wide_att = S.C(*[(n, ("bitlist", 1 << 20) if n == "aggregation_bits" else t) for n, t in S.AttestationElectra[1]])
    wide_idx = S.C(*[(n, ("list", S.U64, 1 << 20) if n == "attesting_indices" else t)
                     for n, t in S.IndexedAttestationElectra[1]])
    dr193 = S.C(*(S.DepositRequest[1] + [("pad", ("bytes", 1))]))
    in_body, in_payload = lambda v: v["body"], lambda v: v["body"]["execution_payload"]
    grow = lambda get, key: (lambda v: get(v)[key].append(get(v)[key][0]))   # one element past the limit
    cases = [   # (label, generator arguments at the limit, the step past it, the field types that can serialise it)
        ("9 attestations", dict(bit_lengths=[10] * 8), grow(in_body, "attestations"),
         dict(body={"attestations": ("list", S.AttestationElectra, 16)})),
        ("2 attester slashings", dict(), grow(in_body, "attester_slashings"),
         dict(body={"attester_slashings": ("list", S.AttesterSlashingElectra, 2)})),
        ("2 consolidations", dict(), grow(in_body, "consolidations"),
         dict(body={"consolidations": ("list", S.SignedConsolidation, 2)})),
        ("131073 aggregation bits", dict(bit_lengths=[131072]),
         lambda v: v["body"]["attestations"][0]["aggregation_bits"].append(True),
         dict(body={"attestations": ("list", wide_att, 8)})),
        ("131073 indices", dict(slashing_indices=131072),
         lambda v: v["body"]["attester_slashings"][0]["attestation_1"]["attesting_indices"].append(1 << 21),
         dict(body={"attester_slashings": ("list", S.C(("attestation_1", wide_idx), ("attestation_2", wide_idx)), 1)})),
        ("8193 deposit requests", dict(n_deposit_requests=8192), grow(in_payload, "deposit_requests"),
         dict(payload={"deposit_requests": ("list", S.DepositRequest, 8193)})),
        ("193-byte deposit requests", dict(n_deposit_requests=3),
         lambda v: [r.update(pad=b"\0") for r in v["body"]["execution_payload"]["deposit_requests"]],
         dict(payload={"deposit_requests": ("list", dr193, 8192)})),
        ("17 withdrawal requests", dict(n_withdrawal_requests=16), grow(in_payload, "withdrawal_requests"),
         dict(payload={"withdrawal_requests": ("list", S.ExecutionLayerWithdrawalRequest, 17)})),
    ]
    out = []
    for label, kw, step, retype in cases:
        v, _ = _block(seed=80, n_transactions=3, bits_per_committee=50, **kw)
        step(v)
        out.append((label, S.serialize(_retyped(**retype), v)))
    _, ssz = _block(seed=81, n_transactions=3, bits_per_committee=50, n_deposit_requests=2, n_withdrawal_requests=2)
    body = 84
    o_at, o_dp = body + _u32(ssz, body + 208), body + _u32(ssz, body + 212)
    att0 = o_at + _u32(ssz, o_at)
    pay = body + _u32(ssz, body + 380)
    o_wd, o_dr, o_wr = (_u32(ssz, pay + k) for k in (508, 528, 532))

    def patched(at, value, nbytes=4):
        b = bytearray(ssz)
        b[at:at + nbytes] = value.to_bytes(nbytes, "little")
        return bytes(b)
    out += [("attestation fixed offset 228", patched(att0, 228)), ("attestation fixed offset 240", patched(att0, 240)),
            ("missing bitlist delimiter", patched(o_dp - 1, 0, 1)),
            ("deposit_requests before withdrawals", patched(pay + 528, o_wd - 44)),
            ("withdrawal_requests before deposit_requests", patched(pay + 532, o_dr - 1)),
            ("withdrawal_requests past the payload", patched(pay + 532, o_wr + 10_000)),
            ("consolidations before blob commitments", patched(body + 392, _u32(ssz, body + 388) - 48))]
    return ssz, out


@pytest.mark.gpu
def test_gpu_electra_rejects_malformed_blocks(gpu):
    from lighthouse_b200 import tree_hash, Lhb200Error
    from lighthouse_b200._ffi import EINVAL
    good, bad = _malformed()
    tree_hash.beacon_block_roots([good], "electra")    # the untouched base block hashes
    for label, b in bad:
        with pytest.raises(Lhb200Error) as e:
            tree_hash.beacon_block_roots([b], "electra")
        assert e.value.code == EINVAL, label
