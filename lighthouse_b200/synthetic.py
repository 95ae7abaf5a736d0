"""Synthetic mainnet-shape inputs (SURVEY.md §8d): BeaconStateDeneb SSZ bytes for the tree-hash path.
Pure byte layout with numpy — no hashing happens here."""
import struct

import numpy as np

DENEB_FIXED = 2736653
BASE_FIXED = 2687377
U64_MAX = (1 << 64) - 1
PENDING_BIT_LENGTHS = (0, 1, 255, 256, 257, 2048)


def validators_ssz(n, rng, pubkeys=None):
    """n x 121-byte Validator records shaped like consensus/types/benches/benches.rs:11-47."""
    v = np.zeros((n, 121), dtype=np.uint8)
    if pubkeys is None:
        v[:, 0:48] = rng.integers(0, 256, size=(n, 48), dtype=np.uint8)
    else:
        v[:, 0:48] = np.frombuffer(pubkeys, dtype=np.uint8).reshape(n, 48)
    idx = np.arange(n, dtype="<u8")
    v[:, 48 + 24:48 + 32] = idx.view(np.uint8).reshape(n, 8)  # H256::from_low_u64_le(i)
    v[:, 80:88] = np.frombuffer(struct.pack("<Q", 32_000_000_000), dtype=np.uint8)
    v[:, 88] = 0
    v[:, 89:105] = 0  # activation_eligibility_epoch = activation_epoch = 0
    v[:, 105:121] = 0xFF  # exit_epoch = withdrawable_epoch = u64::MAX
    return v.tobytes()


def pending_attestation_ssz(rng, n_bits, slot=0):
    """One phase0 PendingAttestation (pending_attestation.rs:25-32) with n_bits seeded aggregation bits: its 148-byte
    fixed part (bitlist offset, AttestationData, inclusion_delay, proposer_index), then the bitlist with its delimiter."""
    bits = np.append(rng.integers(0, 2, size=n_bits).astype(np.uint8), np.uint8(1))
    data = (struct.pack("<QQ", slot, int(rng.integers(0, 64))) + rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()
            + struct.pack("<Q", int(rng.integers(0, 1 << 40))) + rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()
            + struct.pack("<Q", int(rng.integers(0, 1 << 40))) + rng.integers(0, 256, size=32, dtype=np.uint8).tobytes())
    tail = struct.pack("<QQ", int(rng.integers(1, 33)), int(rng.integers(0, 1 << 20)))
    return struct.pack("<I", 148) + data + tail + np.packbits(bits, bitorder="little").tobytes()


def pending_attestations_list_ssz(records):
    """SSZ of a List[PendingAttestation, 4096] from its records' SSZ: the offset table, then the records."""
    out, at = [], 4 * len(records)
    for r in records:
        out.append(struct.pack("<I", at))
        at += len(r)
    return b"".join(out + list(records))


def pending_attestations_ssz(n, rng, bit_lengths=PENDING_BIT_LENGTHS, slot=0):
    """n seeded PendingAttestations, record i with bit_lengths[i % len(bit_lengths)] aggregation bits, as a list."""
    return pending_attestations_list_ssz([pending_attestation_ssz(rng, bit_lengths[i % len(bit_lengths)], slot)
                                          for i in range(n)])


def beacon_state_deneb_ssz(n_validators, seed=1, all_default=False, n_hist_roots=758, n_votes=1024,
                           n_summaries=600, extra_data_len=14, fork="deneb", n_pending=(700, 333, 45),
                           n_pending_attestations=(128, 64), pending_bit_lengths=PENDING_BIT_LENGTHS):
    """SSZ(BeaconState<fork>), mainnet preset; fork in base / altair / bellatrix / capella / deneb / electra
    (beacon_state.rs:224-571: later forks append fields and widen the execution payload header; n_pending = lengths of
    Electra's pending_balance_deposits / pending_partial_withdrawals / pending_consolidations).  Base (phase0) has
    Altair's first 21 fields with previous_ / current_epoch_attestations (n_pending_attestations records, with
    pending_bit_lengths aggregation bits in turn) in place of the participation lists.  all_default=True leaves every
    non-validator field zero so the ZERO_HASHES ladder paths are exercised."""
    base = fork == "base"
    hdr_fixed = {"base": 0, "altair": 0, "bellatrix": 536, "capella": 568, "deneb": 584, "electra": 648}[fork]
    has_tail = fork in ("capella", "deneb", "electra")
    electra = fork == "electra"
    rng = np.random.default_rng(seed)
    V = n_validators

    def rnd(nbytes):
        if all_default:
            return bytes(nbytes)
        return rng.integers(0, 256, size=nbytes, dtype=np.uint8).tobytes()

    if all_default:
        n_hist_roots = n_votes = n_summaries = extra_data_len = 0
        n_pending = (0, 0, 0)
        n_pending_attestations = (0, 0)
    hist = rnd(32 * n_hist_roots)
    votes = rnd(72 * n_votes)
    vals = validators_ssz(V, rng)
    bal = np.arange(V, dtype="<u8").tobytes()
    if all_default:
        pp = bytes(V)
        cp = bytes(V)
        inact = bytes(8 * V)
        slash = bytes(8192 * 8)
    else:
        pp = rng.integers(0, 8, size=V, dtype=np.uint8).tobytes()
        cp = rng.integers(0, 8, size=V, dtype=np.uint8).tobytes()
        inact = rng.integers(0, 64, size=V, dtype="<u8").tobytes()
        slash = rng.integers(0, 1 << 40, size=8192, dtype="<u8").tobytes()
    leph = (rnd(32) + rnd(20) + rnd(32) + rnd(32) + rnd(256) + rnd(32) + rnd(8) + rnd(8) + rnd(8) + rnd(8)
            + struct.pack("<I", hdr_fixed) + rnd(32) + rnd(32) + rnd(32) + rnd(32) + rnd(8) + rnd(8) + rnd(32) + rnd(32))
    leph = (leph[:hdr_fixed] + rnd(extra_data_len)) if hdr_fixed else b""
    assert len(leph) == (hdr_fixed + extra_data_len if hdr_fixed else 0)
    summ = rnd(64 * n_summaries) if has_tail else b""
    pend = [rnd(sz * n) if electra else b"" for sz, n in zip((16, 24, 16), n_pending)]
    fixed_len = DENEB_FIXED - (0 if has_tail else 20) - (0 if hdr_fixed else 4) + (60 if electra else 0)
    if base:   # the pending-attestation lists take the participation lists' places; nothing after the checkpoints
        pp, cp = (pending_attestations_ssz(n, rng, pending_bit_lengths) for n in n_pending_attestations)
        inact = b""
        fixed_len = BASE_FIXED

    o_hist = fixed_len
    o_votes = o_hist + len(hist)
    o_val = o_votes + len(votes)
    o_bal = o_val + len(vals)
    o_pp = o_bal + len(bal)
    o_cp = o_pp + len(pp)
    o_inact = o_cp + len(cp)
    o_leph = o_inact + len(inact)
    o_hs = o_leph + len(leph)
    o_pbd = o_hs + len(summ)
    o_ppw = o_pbd + len(pend[0])
    o_pc = o_ppw + len(pend[1])
    u32 = lambda x: struct.pack("<I", x)
    fixed = b"".join([
        rnd(8), rnd(32), rnd(8),                       # genesis_time, genesis_validators_root, slot
        rnd(16),                                       # fork
        rnd(112),                                      # latest_block_header
        rnd(8192 * 32), rnd(8192 * 32),                # block_roots, state_roots
        u32(o_hist), rnd(72), u32(o_votes), rnd(8),    # historical_roots, eth1_data, eth1_data_votes, deposit idx
        u32(o_val), u32(o_bal),
        rnd(65536 * 32), slash,                        # randao_mixes, slashings
        u32(o_pp), u32(o_cp),
        bytes([0 if all_default else 0x0B]),           # justification_bits
        rnd(40), rnd(40), rnd(40),                     # checkpoints
    ])
    if not base:   # Altair on: inactivity scores, sync committees, then what later forks append
        fixed += b"".join([
            u32(o_inact),
            (vals[:48] * 1 if False else rnd(513 * 48)),   # current_sync_committee (512 pubkeys + aggregate)
            rnd(513 * 48),                                 # next_sync_committee
            (u32(o_leph) if hdr_fixed else b""), ((rnd(8) + rnd(8) + u32(o_hs)) if has_tail else b""),
            ((rnd(48) + u32(o_pbd) + u32(o_ppw) + u32(o_pc)) if electra else b""),   # six u64s, three list offsets
        ])
    assert len(fixed) == fixed_len, len(fixed)
    return b"".join([fixed, hist, votes, vals, bal, pp, cp, inact, leph, summ] + pend)


# ---------------------------------------------------------------------------------------------------------
# Synthetic attestation SignatureSets (SURVEY.md §8d).  Secret keys are the interop keys
# (common/eth2_interop_keypairs/src/lib.rs:40-56); public keys and signatures are produced by the CUDA
# library's own sk_to_pk / sign kernels (the SecretKey surface), so this module has no curve arithmetic.
CURVE_ORDER = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
MAINNET_GVR = bytes.fromhex("4b363db94e286120d76eb905340fdd4e54bfe9f06bf33ff6cf5ad27f511bfe95")


def interop_secret_keys(n):
    import hashlib
    out = []
    for i in range(n):
        out.append(int.from_bytes(hashlib.sha256(i.to_bytes(32, "little")).digest(), "little") % CURVE_ORDER)
    return out


def _sha(b):
    import hashlib
    return hashlib.sha256(b).digest()


def attester_domain(fork_version=bytes.fromhex("04000000"), gvr=MAINNET_GVR):
    """compute_domain(DOMAIN_BEACON_ATTESTER = 1, fork_version, genesis_validators_root) (chain_spec.rs:548-566)"""
    fork_data_root = _sha(fork_version + bytes(28) + gvr)
    return (1).to_bytes(4, "little") + fork_data_root[:28]


def attestation_signing_root(j, epoch, domain):
    """signing_root(AttestationData{slot, index, beacon_block_root, source, target}, domain)
    (attestation_data.rs:28-39, signing_data.rs:27-35).  Synthetic field values per SURVEY §8d."""
    u64 = lambda v: v.to_bytes(8, "little") + bytes(24)
    slot = (j // 64) % 32 + 32 * epoch
    bbr = _sha(b"bbr" + j.to_bytes(8, "little"))
    src = _sha(u64(epoch - 1) + _sha(b"src"))
    tgt = _sha(u64(epoch) + _sha(b"tgt"))
    z = bytes(32)
    l1 = [_sha(u64(slot) + u64(j % 64)), _sha(bbr + src), _sha(tgt + z), _sha(z + z)]
    root = _sha(_sha(l1[0] + l1[1]) + _sha(l1[2] + l1[3]))
    return _sha(root + domain)


class AttestationBatch:
    """SoA buffers for lhb200_verify_signature_sets."""

    def __init__(self, sigs, msgs, pks, offsets, committees, pk_table):
        self.sigs, self.msgs, self.pks, self.offsets = sigs, msgs, pks, offsets
        self.committees, self.pk_table = committees, pk_table
        self.n_sets = len(offsets) - 1

    @property
    def input_bytes(self):
        return len(self.sigs) + len(self.msgs) + len(self.pks) + 8 * self.n_sets


def sets_workload(key_counts, n_validators=16384, seed=0x11570000, epoch=100, first_index=0):
    """The DEFINITION of a synthetic batch of SignatureSets, without any curve arithmetic (numpy + hashlib only, so the
    CPU reference arm of bench.py builds the very same workload without loading the CUDA library):
    set j (global index first_index + j) is signed by key_counts[j] distinct validators perm[(a_j + t b_j) mod V]
    (b_j odd, V a power of two) over the attestation signing root of its global index (SURVEY.md §8d).
    -> dict(committees uint32[K], offsets uint32[n+1], agg_sk list[int] (sum of the signers' interop keys mod r),
            msgs bytes n*32, n_validators)"""
    key_counts = np.asarray(key_counts, dtype=np.int64)
    n_sets = len(key_counts)
    V = n_validators
    assert V & (V - 1) == 0 and int(key_counts.max(initial=0)) <= V
    rng = np.random.default_rng(seed)
    perm = rng.permutation(V)
    # a_j, b_j are functions of the GLOBAL set index, so a shard [first_index, first_index + n) of a larger batch is
    # generated exactly as the same range of the whole batch
    gidx = np.arange(first_index, first_index + n_sets, dtype=np.uint64)
    mix = (gidx * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    a = (mix >> np.uint64(7)) % np.uint64(V)
    b = ((mix >> np.uint64(29)) % np.uint64(V // 2)) * np.uint64(2) + np.uint64(1)
    offsets = np.zeros(n_sets + 1, dtype=np.uint64)
    np.cumsum(key_counts, out=offsets[1:])
    K = int(offsets[-1])
    set_of_key = np.repeat(np.arange(n_sets), key_counts)
    t = np.arange(K, dtype=np.uint64) - offsets[:-1][set_of_key]
    committees = perm[((a[set_of_key] + t * b[set_of_key]) % np.uint64(V)).astype(np.int64)].astype(np.uint32)
    sks = interop_secret_keys(V)
    words = np.array([[(s >> (32 * w)) & 0xFFFFFFFF for w in range(8)] for s in sks], dtype=np.uint64)
    agg = []
    CH = 1 << 20
    sums = np.zeros((n_sets, 8), dtype=np.uint64)
    # limb-wise sums (8 x 32-bit words held in uint64), recombined with Python ints
    if n_sets and np.all(key_counts == key_counts[0]) and key_counts[0] > 0:
        k = int(key_counts[0])
        rows = max(1, CH // k)
        for lo in range(0, n_sets, rows):
            hi = min(n_sets, lo + rows)
            sums[lo:hi] = words[committees[lo * k:hi * k].reshape(hi - lo, k)].sum(axis=1)
    else:
        for lo in range(0, K, CH):
            hi = min(K, lo + CH)
            np.add.at(sums, set_of_key[lo:hi], words[committees[lo:hi]])
    for row in sums:
        v = 0
        for w in range(8):
            v += int(row[w]) << (32 * w)
        agg.append(v % CURVE_ORDER)
    domain = attester_domain()
    msgs = b"".join(attestation_signing_root(first_index + j, epoch, domain) for j in range(n_sets))
    return {"committees": committees, "offsets": offsets.astype(np.uint32), "agg_sk": agg, "msgs": msgs,
            "n_validators": V, "sks": sks}


def materialize_sets(work, pk_table96, sign_fn):
    """Attach keys and signatures to a sets_workload(): pk_table96 = uint8[V, 96] uncompressed keys of the interop
    validators, sign_fn(sk_bytes n*32, msgs n*32) -> n*96 compressed signatures (the CUDA library's lhb200_sign for the
    GPU arm, the CPU oracle for the reference arm)."""
    sigs = sign_fn(b"".join(v.to_bytes(32, "big") for v in work["agg_sk"]), work["msgs"])
    pks = pk_table96[work["committees"]].tobytes()
    n = len(work["offsets"]) - 1
    offs = work["offsets"]
    comm = work["committees"]
    if n and np.all(np.diff(offs) == np.diff(offs)[0]):
        comm = comm.reshape(n, -1)
    return AttestationBatch(sigs, work["msgs"], pks, offs, comm, pk_table96)


def interop_pubkey_table(n_validators):
    """uint8[V, 96]: uncompressed interop public keys, produced by the CUDA library's sk_to_pk kernel."""
    from . import bls
    sk_bytes = b"".join(s.to_bytes(32, "big") for s in interop_secret_keys(n_validators))
    _, pk96 = bls.sk_to_pk(sk_bytes)
    return np.frombuffer(pk96, dtype=np.uint8).reshape(n_validators, 96)


def attestation_batch(n_sets, keys_per_set=128, n_validators=16384, seed=0x11570000, epoch=100, first_index=0,
                      pk_table=None):
    """n_sets aggregate attestations, each signed by `keys_per_set` distinct validators.  Needs lhb200.init()."""
    from . import bls
    work = sets_workload(np.full(n_sets, keys_per_set), n_validators, seed, epoch, first_index)
    if pk_table is None:
        pk_table = interop_pubkey_table(n_validators)
    return materialize_sets(work, pk_table, bls.sign)


def block_signature_key_counts(n_blocks=32, n_validators=524288):
    """Key counts of the SignatureSets a full Deneb block contributes to BlockSignatureVerifier
    (block_signature_verifier.rs:141-171, SURVEY.md §8d cfg3): proposal, randao, 128 attestations (committee =
    V / 32 / 64 keys), the sync aggregate (512 keys), 16 exits, 16 BLS-to-execution changes."""
    committee = max(1, n_validators // 32 // 64)
    per_block = [1, 1] + [committee] * 128 + [512] + [1] * 16 + [1] * 16
    return np.array(per_block * n_blocks, dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------
# Synthetic Deneb BeaconBlock (mainnet preset) — values + SSZ bytes (SURVEY §8 a15).
def beacon_block_deneb(seed=1, n_attestations=128, n_transactions=150, n_proposer_slashings=1,
                       n_attester_slashings=1, n_deposits=2, n_exits=3, n_bls_changes=4, n_withdrawals=16,
                       n_blobs=6, tx_sizes=None, committee=244, extra_data_len=13, fork="deneb"):
    """-> (value, ssz_bytes) of a BeaconBlock<fork> (base / altair / bellatrix / capella / deneb: the later forks' fields
    are dropped, beacon_block_body.rs:33-110; Base has no sync_aggregate) filled with seeded pseudo-random content of
    mainnet shape."""
    from . import ssz_schema as S
    rng = np.random.default_rng(seed)

    def rb(n):
        return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()

    def u64():
        return int(rng.integers(0, 1 << 62))

    def checkpoint():
        return {"epoch": u64(), "root": rb(32)}

    def att_data():
        return {"slot": u64(), "index": u64() % 64, "beacon_block_root": rb(32), "source": checkpoint(),
                "target": checkpoint()}

    def header():
        return {"message": {"slot": u64(), "proposer_index": u64(), "parent_root": rb(32), "state_root": rb(32),
                            "body_root": rb(32)}, "signature": rb(96)}

    def indexed(n):
        return {"attesting_indices": sorted(int(x) for x in rng.integers(0, 1 << 20, size=n)), "data": att_data(),
                "signature": rb(96)}

    if tx_sizes is None:
        # mainnet-like mix: mostly a few hundred bytes, some multi-KB calldata, the odd empty / chunk-boundary size
        tx_sizes = [int(x) for x in rng.choice([0, 1, 31, 32, 33, 110, 180, 256, 257, 700, 2_500, 20_000],
                                               size=n_transactions)]
    payload = {
        "parent_hash": rb(32), "fee_recipient": rb(20), "state_root": rb(32), "receipts_root": rb(32),
        "logs_bloom": rb(256), "prev_randao": rb(32), "block_number": u64(), "gas_limit": 30_000_000,
        "gas_used": u64() % 30_000_000, "timestamp": u64(), "extra_data": rb(extra_data_len),
        "base_fee_per_gas": int.from_bytes(rb(12), "little"), "block_hash": rb(32),
        "transactions": [rb(n) for n in tx_sizes],
        "withdrawals": [{"index": u64(), "validator_index": u64(), "address": rb(20), "amount": u64()}
                        for _ in range(n_withdrawals)],
        "blob_gas_used": 131072 * n_blobs, "excess_blob_gas": u64()}
    body = {
        "randao_reveal": rb(96),
        "eth1_data": {"deposit_root": rb(32), "deposit_count": u64(), "block_hash": rb(32)},
        "graffiti": rb(32),
        "proposer_slashings": [{"signed_header_1": header(), "signed_header_2": header()}
                               for _ in range(n_proposer_slashings)],
        "attester_slashings": [{"attestation_1": indexed(committee), "attestation_2": indexed(committee // 2 + 1)}
                               for _ in range(n_attester_slashings)],
        "attestations": [{"aggregation_bits": [bool(b) for b in rng.integers(0, 2, size=min(2048, committee + (i % 7)))],
                          "data": att_data(), "signature": rb(96)} for i in range(n_attestations)],
        "deposits": [{"proof": [rb(32) for _ in range(33)],
                      "data": {"pubkey": rb(48), "withdrawal_credentials": rb(32), "amount": 32_000_000_000,
                               "signature": rb(96)}} for _ in range(n_deposits)],
        "voluntary_exits": [{"message": {"epoch": u64(), "validator_index": u64()}, "signature": rb(96)}
                            for _ in range(n_exits)],
        "sync_aggregate": {"sync_committee_bits": [bool(b) for b in rng.integers(0, 2, size=512)],
                           "sync_committee_signature": rb(96)},
        "execution_payload": payload,
        "bls_to_execution_changes": [{"message": {"validator_index": u64(), "from_bls_pubkey": rb(48),
                                                  "to_execution_address": rb(20)}, "signature": rb(96)}
                                     for _ in range(n_bls_changes)],
        "blob_kzg_commitments": [rb(48) for _ in range(n_blobs)]}
    block = {"slot": u64(), "proposer_index": u64() % 500_000, "parent_root": rb(32), "state_root": rb(32),
             "body": body}
    if fork != "deneb":
        body_t = S.BEACON_BLOCK_BODY_BY_FORK[fork]
        if fork not in ("base", "altair"):
            pt = S.EXECUTION_PAYLOAD_BY_FORK[fork]
            body["execution_payload"] = {n: payload[n] for n, _ in pt[1]}
        block["body"] = {n: body[n] for n, _ in body_t[1]}
    return block, S.serialize(S.BEACON_BLOCK_BY_FORK[fork], block)


def blind_block_deneb(block, transactions_root: bytes, withdrawals_root: bytes, fork="deneb"):
    """BlindedBeaconBlock<fork> value + SSZ of `block` (as produced by beacon_block_deneb) given the two list roots
    of its payload (computed by whoever has a hasher: the CUDA library, the oracle or the spec restatement)."""
    import copy
    from . import ssz_schema as S
    v = copy.deepcopy(block)
    p = v["body"]["execution_payload"]
    hdr = {k: p[k] for k in p if k not in ("transactions", "withdrawals")}
    hdr["transactions_root"], hdr["withdrawals_root"] = transactions_root, withdrawals_root
    v["body"]["execution_payload"] = {n: hdr[n] for n, _ in S.EXECUTION_PAYLOAD_HEADER_BY_FORK[fork][1]}
    return v, S.serialize(S.BLINDED_BEACON_BLOCK_BY_FORK[fork], v)


# ---------------------------------------------------------------------------------------------------------
# Synthetic Electra BeaconBlock (mainnet preset, beacon_block_body.rs:70-121).  A generator of its own, so the Deneb
# generator above keeps its exact byte output (and random stream) for every existing caller.
def beacon_block_electra(seed=1, n_attestations=8, committees_per_attestation=4, bits_per_committee=500,
                         n_deposit_requests=4, n_withdrawal_requests=16, n_consolidations=1, n_attester_slashings=1,
                         slashing_indices=None, bit_lengths=None, **deneb_kw):
    """-> (value, ssz_bytes) of a BeaconBlockElectra.  The fields Electra shares with Deneb come from
    beacon_block_deneb(seed, **deneb_kw); the Electra operations from a second seeded stream.  Attestation i covers
    `committees_per_attestation` committees (committee_bits) of `bits_per_committee` + i % 7 aggregation bits, unless
    `bit_lengths` gives every attestation's bit count (n_attestations is then len(bit_lengths)).  The first indexed
    attestation of each attester slashing has `slashing_indices` indices (default: one attestation's bit count)."""
    from . import ssz_schema as S
    block, _ = beacon_block_deneb(seed=seed, n_attestations=0, n_attester_slashings=0, **deneb_kw)
    rng = np.random.default_rng([seed, 5])

    def rb(n):
        return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()

    def u64():
        return int(rng.integers(0, 1 << 62))

    def att_data():  # Electra: the committee index moved to committee_bits, data.index is 0
        cp = lambda: {"epoch": u64(), "root": rb(32)}
        return {"slot": u64(), "index": 0, "beacon_block_root": rb(32), "source": cp(), "target": cp()}

    def indexed(n):
        return {"attesting_indices": sorted(int(x) for x in rng.integers(0, 1 << 20, size=n)), "data": att_data(),
                "signature": rb(96)}

    k = min(64, committees_per_attestation)
    if bit_lengths is None:
        bit_lengths = [k * bits_per_committee + i % 7 for i in range(n_attestations)]
    if slashing_indices is None:
        slashing_indices = k * bits_per_committee
    attestations = []
    for nb in bit_lengths:
        committees = {int(c) for c in rng.choice(64, size=k, replace=False)}
        attestations.append({"aggregation_bits": rng.integers(0, 2, size=nb).astype(bool).tolist(), "data": att_data(),
                             "committee_bits": [c in committees for c in range(64)], "signature": rb(96)})
    body = block["body"]
    body["attester_slashings"] = [{"attestation_1": indexed(slashing_indices),
                                   "attestation_2": indexed(slashing_indices // 2 + 1)} for _ in range(n_attester_slashings)]
    body["attestations"] = attestations
    body["execution_payload"]["deposit_requests"] = [
        {"pubkey": rb(48), "withdrawal_credentials": rb(32), "amount": u64(), "signature": rb(96), "index": u64()}
        for _ in range(n_deposit_requests)]
    body["execution_payload"]["withdrawal_requests"] = [
        {"source_address": rb(20), "validator_pubkey": rb(48), "amount": u64()} for _ in range(n_withdrawal_requests)]
    body["consolidations"] = [{"message": {"source_index": u64(), "target_index": u64(), "epoch": u64()},
                               "signature": rb(96)} for _ in range(n_consolidations)]
    return block, S.serialize(S.BEACON_BLOCK_BY_FORK["electra"], block)


def blind_block_electra(block, transactions_root: bytes, withdrawals_root: bytes, deposit_requests_root: bytes,
                        withdrawal_requests_root: bytes):
    """BlindedBeaconBlockElectra value + SSZ of `block` (as produced by beacon_block_electra) given the four list roots
    of its payload (ExecutionPayloadHeaderElectra, execution_payload_header.rs:88-93)."""
    import copy
    from . import ssz_schema as S
    v = copy.deepcopy(block)
    p = v["body"]["execution_payload"]
    hdr = {k: p[k] for k in p if k not in ("transactions", "withdrawals", "deposit_requests", "withdrawal_requests")}
    hdr.update(transactions_root=transactions_root, withdrawals_root=withdrawals_root,
               deposit_requests_root=deposit_requests_root, withdrawal_requests_root=withdrawal_requests_root)
    v["body"]["execution_payload"] = {n: hdr[n] for n, _ in S.ExecutionPayloadHeaderElectra[1]}
    return v, S.serialize(S.BLINDED_BEACON_BLOCK_BY_FORK["electra"], v)


# ---------------------------------------------------------------------------------------------------------
# Signed Attestations over a committee cache (lhb200_attestations_verify, lighthouse_b200.attestations).  Validator i
# holds interop key i (interop_pubkey_table); an attestation is signed by (sum of its attesters' secret keys mod r) .
# H(signing root) through the CUDA library's lhb200_sign, which is the aggregate of the attesters' own signatures.
def attestation_data_ssz(slot, index, beacon_block_root, source, target):
    """AttestationData {slot, index, beacon_block_root, source: (epoch, root), target: (epoch, root)}: 128 bytes."""
    return (struct.pack("<QQ", slot, index) + beacon_block_root + struct.pack("<Q", source[0]) + source[1]
            + struct.pack("<Q", target[0]) + target[1])


def attestation_data_root(data):
    """hash_tree_root(AttestationData): 8 leaves, the checkpoints as 2-leaf containers."""
    def leaf(b):
        return b + bytes(32 - len(b))
    z = bytes(32)
    l0 = _sha(_sha(leaf(data[0:8]) + leaf(data[8:16])) + _sha(data[16:48] + _sha(leaf(data[48:56]) + data[56:88])))
    l1 = _sha(_sha(_sha(leaf(data[88:96]) + data[96:128]) + z) + _sha(z + z))
    return _sha(l0 + l1)


def attestation_ssz(bits, data, signature, committee_bits=None):
    """SSZ of an Attestation: Base to Deneb {aggregation_bits: Bitlist[2048], data, signature}, or with committee_bits
    (an int, Bitvector[64]) Electra's {aggregation_bits: Bitlist[131072], data, signature, committee_bits}."""
    bits = np.append(np.asarray(bits, dtype=np.uint8), np.uint8(1))
    tail = b"" if committee_bits is None else struct.pack("<Q", committee_bits)
    fixed = 228 + len(tail)
    return struct.pack("<I", fixed) + data + signature + tail + np.packbits(bits, bitorder="little").tobytes()


ATTESTATION_KINDS = ("unaggregated", "aggregate", "electra")


def signed_attestations(cache, kind, n, sks, fork_info, gvr=MAINNET_GVR, seed=0, slot=None, n_committees=2,
                        committees_per_attestation=4, fill=1.0):
    """n signed Attestations over a committees.CommitteeCache whose validators hold the interop keys `sks`
    (interop_secret_keys), signed for fork_info = (previous_version, current_version, fork epoch) and gvr.
      unaggregated  one bit each, at `slot` (default the epoch's first), over n_committees committees of that slot:
                    attestation j is committee j % n_committees, member j // n_committees; the attestations of one
                    committee share their AttestationData, as gossip does.
      aggregate     attestation j is committee j % committees_per_slot of slot epoch_start + (j // committees_per_slot)
                    % 32, with `fill` of its bits set (1.0: all).
      electra       Electra: attestation j covers committees_per_attestation consecutive committees (mod
                    committees_per_slot) of slot epoch_start + j % 32 in committee_bits, with `fill` of the bits set.
    The target epoch is the cache's, so fork_info's epoch picks the version.  Needs lighthouse_b200.init()."""
    from . import bls
    assert kind in ATTESTATION_KINDS
    rng = np.random.default_rng(seed)
    epoch = cache.initialized_epoch
    start = epoch * 32
    cps = cache.committees_per_slot()
    prev, cur, fork_epoch = fork_info
    domain = attester_domain(bytes(prev) if epoch < fork_epoch else bytes(cur), gvr)
    source = (max(epoch - 1, 0), _sha(b"source" + struct.pack("<QQ", seed, epoch)))
    target = (epoch, _sha(b"target" + struct.pack("<QQ", seed, epoch)))
    records = []   # (bits, data, committee_bits or None, attesters)
    for j in range(n):
        if kind == "unaggregated":
            s = start if slot is None else slot
            index = (j % n_committees) % cps
            members = cache.get_beacon_committee(s, index).committee
            bits = np.zeros(len(members), dtype=np.uint8)
            if len(members):
                bits[(j // n_committees) % len(members)] = 1
            bbr = _sha(b"head" + struct.pack("<QQQ", seed, s, index))
            records.append((bits, attestation_data_ssz(s, index, bbr, source, target), None, members[bits == 1]))
            continue
        if kind == "aggregate":
            s, indices = start + (j // cps) % 32, [j % cps]
        else:
            k = min(committees_per_attestation, cps)
            s, indices = start + j % 32, sorted({(j * k + t) % cps for t in range(k)})
        members = np.concatenate([cache.get_beacon_committee(s, c).committee for c in indices])
        bits = (rng.random(len(members)) < fill).astype(np.uint8)
        if len(members) and not bits.any():
            bits[int(rng.integers(0, len(members)))] = 1
        bbr = _sha(b"head" + struct.pack("<QQ", seed, j))
        data = attestation_data_ssz(s, 0 if kind == "electra" else indices[0], bbr, source, target)
        cbits = sum(1 << c for c in indices) if kind == "electra" else None
        records.append((bits, data, cbits, members[bits == 1]))
    # (an attestation without attesters is signed with key 1: its set has no keys and fails with status 4 anyway)
    agg = [sum(sks[int(v)] for v in attesters) % CURVE_ORDER or 1 for _, _, _, attesters in records]
    msgs = b"".join(_sha(attestation_data_root(data) + domain) for _, data, _, _ in records)
    sigs = bls.sign(b"".join(a.to_bytes(32, "big") for a in agg), msgs)
    return [attestation_ssz(bits, data, sigs[96 * j:96 * j + 96], cbits)
            for j, (bits, data, cbits, _) in enumerate(records)]


# ---------------------------------------------------------------------------------------------------------
# Signed blocks over a resident world (lhb200_block_signatures_verify, lighthouse_b200.block_signatures).  Validator i
# holds interop key i; every signature is (sum of its signers' secret keys mod r) . H(signing root) from `sign_fn`
# (default: the CUDA library's lhb200_sign), which is the aggregate of the signers' own signatures.
O_STATE_GVR, O_STATE_SLOT, O_STATE_FORK, O_STATE_VAL_OFF, O_STATE_CSC = 8, 40, 48, 524552, 2687381
DOMAIN_PROPOSER, DOMAIN_ATTESTER, DOMAIN_RANDAO, DOMAIN_EXIT, DOMAIN_SYNC = 0, 1, 2, 4, 7
DOMAIN_BLS_TO_EXECUTION_CHANGE, DOMAIN_CONSOLIDATION = 0x0A, 0x0B
INFINITY_SIGNATURE = b"\xc0" + bytes(95)


def compute_domain(domain_type, version, gvr):
    return domain_type.to_bytes(4, "little") + _sha(bytes(version) + bytes(28) + bytes(gvr))[:28]


def _chunk(v):
    return struct.pack("<Q", v) + bytes(24)


def header_root(slot, proposer_index, parent_root, state_root, body_root):
    z = bytes(32)
    return _sha(_sha(_sha(_chunk(slot) + _chunk(proposer_index)) + _sha(parent_root + state_root))
                + _sha(_sha(body_root + z) + _sha(z + z)))


def g1_compress(pk96):
    """48-byte compressed form of a 96-byte uncompressed G1 point (x || y, big-endian; not infinity)."""
    p = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
    y = int.from_bytes(pk96[48:], "big")
    out = bytearray(pk96[:48])
    out[0] |= 0x80 | (0x20 if y > (p - 1) // 2 else 0)
    return bytes(out)


def block_signature_state(n, fork, slot, fork_versions, pubkeys48, sync_members=None, seed=5):
    """SSZ of a BeaconState<fork> of n validators at `slot` whose records carry `pubkeys48` (n x 48 bytes, validator i's
    compressed key), whose fork is fork_versions = (previous_version, current_version, epoch), and whose
    current_sync_committee names `sync_members` (512 validator indices; default 7919 i mod n)."""
    ssz = bytearray(beacon_state_deneb_ssz(n, seed=seed, fork=fork, n_votes=3, n_hist_roots=5, n_summaries=2))
    struct.pack_into("<Q", ssz, O_STATE_SLOT, slot)
    prev, cur, epoch = fork_versions
    ssz[O_STATE_FORK:O_STATE_FORK + 16] = bytes(prev) + bytes(cur) + struct.pack("<Q", epoch)
    lo = struct.unpack_from("<I", ssz, O_STATE_VAL_OFF)[0]
    v = np.frombuffer(ssz, dtype=np.uint8, count=121 * n, offset=lo).reshape(n, 121)
    v[:, :48] = np.frombuffer(bytes(pubkeys48), dtype=np.uint8).reshape(n, 48)
    if fork != "base":
        if sync_members is None:
            sync_members = [(7919 * i) % n for i in range(512)]
        pk = np.frombuffer(bytes(pubkeys48), dtype=np.uint8).reshape(n, 48)
        ssz[O_STATE_CSC:O_STATE_CSC + 512 * 48] = pk[np.asarray(sync_members, dtype=np.int64)].tobytes()
    return bytes(ssz)


def _attestation_value(ssz, electra):
    """Attestation SSZ in lhb200_attestations_verify's layout -> the block body's value"""
    data = ssz[4:132]
    fixed = 236 if electra else 228
    raw = np.frombuffer(ssz[fixed:], dtype=np.uint8)
    bits = np.unpackbits(raw, bitorder="little")[:8 * (len(raw) - 1) + int(raw[-1]).bit_length() - 1]
    s, i, bbr, se, sr, te, tr = struct.unpack_from("<QQ32sQ32sQ32s", data)
    v = {"aggregation_bits": [bool(b) for b in bits], "signature": ssz[132:228],
         "data": {"slot": s, "index": i, "beacon_block_root": bbr, "source": {"epoch": se, "root": sr},
                  "target": {"epoch": te, "root": tr}}}
    if electra:
        cb = struct.unpack_from("<Q", ssz, 228)[0]
        v["committee_bits"] = [bool((cb >> k) & 1) for k in range(64)]
    return v


def signed_beacon_block(fork, slot, proposer, sks, state_fork, gvr, versions, block_root_fn, sign_fn=None, seed=0,
                        attestations=(), n_proposer_slashings=1, n_attester_slashings=1, slashing_size=3,
                        n_exits=2, sync_committee=None, sync_participation=0.9, n_consolidations=None,
                        n_validators=None, n_bls_changes=None, bls_change_pubkeys=None, pk_fn=None):
    """-> (SignedBeaconBlock SSZ, block root) of a BeaconBlock<fork> at `slot` by `proposer`, every set signed with the
    interop keys `sks`: the proposal (over block_root_fn(BeaconBlock SSZ)), the RANDAO reveal, n proposer and attester
    slashings (slashing_size signers each), `attestations` (SSZ in lhb200_attestations_verify's layout, e.g.
    signed_attestations), n exits, the sync aggregate over `sync_committee` (its 512 validator indices) with
    `sync_participation` of the bits set (0: all zero, with the infinity signature), from Capella n BLS-to-execution
    changes (2 by default) signed by keys outside the registry (`bls_change_pubkeys` replaces their from_bls_pubkey
    bytes, for keys that must fail to decode; pk_fn(sk bytes) -> compressed keys, default the CUDA library's
    lhb200_sk_to_pk), and Electra's consolidations (1 by default).  state_fork = (previous_version, current_version, epoch); versions = (genesis_fork_version,
    capella_fork_version).  Deposits (2) carry no set.  Bellatrix on, the payload has 4 small transactions."""
    from . import ssz_schema as S
    if sign_fn is None:
        from . import bls
        sign_fn = bls.sign
    rng = np.random.default_rng([seed, slot, 11])
    n_val = n_validators or len(sks)
    electra, epoch = fork == "electra", slot // 32
    prev, cur, fork_epoch = state_fork

    def domain(dtype, e):
        return compute_domain(dtype, prev if e < fork_epoch else cur, gvr)

    def rb(n):
        return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()

    def pick(k):
        return sorted(int(x) for x in rng.choice(n_val, size=k, replace=False))

    todo = []   # (signers, signing root, setter)

    def signed(signers, root, setter):
        todo.append((signers, root, setter))

    if electra:
        block, _ = beacon_block_electra(seed=seed + 1, n_attestations=0, n_attester_slashings=0, n_consolidations=0,
                                        n_deposit_requests=1, n_withdrawal_requests=1, n_transactions=4, n_exits=0,
                                        n_bls_changes=0, n_proposer_slashings=0, n_deposits=2)
    else:
        block, _ = beacon_block_deneb(seed=seed + 1, n_attestations=0, n_transactions=4, n_proposer_slashings=0,
                                      n_attester_slashings=0, n_deposits=2, n_exits=0, n_bls_changes=0, fork=fork)
    body = block["body"]
    block.update(slot=slot, proposer_index=proposer, parent_root=_sha(b"parent" + struct.pack("<QQ", seed, slot)))
    signed([proposer], _sha(_chunk(epoch) + domain(DOMAIN_RANDAO, epoch)), lambda s: body.update(randao_reveal=s))
    body["proposer_slashings"] = []
    for j in range(n_proposer_slashings):
        v, hs = pick(1)[0], int(rng.integers(0, slot + 1))
        ps = {}
        for k in (1, 2):
            h = {"slot": hs, "proposer_index": v, "parent_root": rb(32), "state_root": rb(32), "body_root": rb(32)}
            root = header_root(hs, v, h["parent_root"], h["state_root"], h["body_root"])
            ps["signed_header_%d" % k] = {"message": h, "signature": None}
            signed([v], _sha(root + domain(DOMAIN_PROPOSER, hs // 32)),
                   lambda s, d=ps["signed_header_%d" % k]: d.update(signature=s))
        body["proposer_slashings"].append(ps)
    body["attester_slashings"] = []
    for j in range(n_attester_slashings):
        sl = {}
        for k in (1, 2):
            idx = pick(slashing_size)
            data = attestation_data_ssz(max(slot - 1, 0), 0, rb(32), (max(epoch - 1, 0), rb(32)), (epoch, rb(32)))
            s_, i_, bbr, se, sr, te, tr = struct.unpack_from("<QQ32sQ32sQ32s", data)
            sl["attestation_%d" % k] = {"attesting_indices": idx, "signature": None, "data": {
                "slot": s_, "index": i_, "beacon_block_root": bbr, "source": {"epoch": se, "root": sr},
                "target": {"epoch": te, "root": tr}}}
            signed(idx, _sha(attestation_data_root(data) + domain(DOMAIN_ATTESTER, te)),
                   lambda s, d=sl["attestation_%d" % k]: d.update(signature=s))
        body["attester_slashings"].append(sl)
    body["attestations"] = [_attestation_value(a, electra) for a in attestations]
    body["voluntary_exits"] = []
    for j in range(n_exits):
        v, e = pick(1)[0], int(rng.integers(0, epoch + 1))
        ex = {"message": {"epoch": e, "validator_index": v}, "signature": None}
        d = compute_domain(DOMAIN_EXIT, versions[1], gvr) if fork in ("deneb", "electra") else domain(DOMAIN_EXIT, e)
        signed([v], _sha(_sha(_chunk(e) + _chunk(v)) + d), lambda s, x=ex: x.update(signature=s))
        body["voluntary_exits"].append(ex)
    if fork != "base":
        bits = [False] * 512
        if sync_participation > 0:
            bits = [bool(b) for b in rng.random(512) < sync_participation]
        body["sync_aggregate"] = {"sync_committee_bits": bits, "sync_committee_signature": INFINITY_SIGNATURE}
        if any(bits):
            prev_slot = max(slot, 1) - 1
            signers = [int(sync_committee[m]) for m in range(512) if bits[m]]
            signed(signers, _sha(block["parent_root"] + domain(DOMAIN_SYNC, prev_slot // 32)),
                   lambda s: body["sync_aggregate"].update(sync_committee_signature=s))
    if fork in ("capella", "deneb", "electra"):
        if pk_fn is None:
            from . import bls
            pk_fn = lambda b: bls.sk_to_pk(b)[0]
        n_ch = 2 if n_bls_changes is None else n_bls_changes
        csks = [int.from_bytes(_sha(b"bls-change" + struct.pack("<QQQ", seed, slot, j)), "little") % CURVE_ORDER
                for j in range(n_ch)]
        pks = pk_fn(b"".join(k.to_bytes(32, "big") for k in csks)) if n_ch else b""
        body["bls_to_execution_changes"] = []
        for j in range(n_ch):
            pk = pks[48 * j:48 * j + 48] if bls_change_pubkeys is None else bls_change_pubkeys[j]
            v, addr = pick(1)[0], rb(20)
            ch = {"message": {"validator_index": v, "from_bls_pubkey": pk, "to_execution_address": addr},
                  "signature": None}
            root = _sha(_sha(_chunk(v) + _sha(pk[:32] + pk[32:] + bytes(16))) + _sha(addr + bytes(12) + bytes(32)))
            todo.append((None, _sha(root + compute_domain(DOMAIN_BLS_TO_EXECUTION_CHANGE, versions[0], gvr)),
                         lambda s, x=ch: x.update(signature=s), csks[j]))
            body["bls_to_execution_changes"].append(ch)
    if electra:
        body["consolidations"] = []
        for j in range(1 if n_consolidations is None else n_consolidations):
            src, tgt = pick(2)
            e = int(rng.integers(0, epoch + 1))
            c = {"message": {"source_index": src, "target_index": tgt, "epoch": e}, "signature": None}
            root = _sha(_sha(_chunk(src) + _chunk(tgt)) + _sha(_chunk(e) + bytes(32)))
            signed([src, tgt], _sha(root + compute_domain(DOMAIN_CONSOLIDATION, versions[0], gvr)),
                   lambda s, x=c: x.update(signature=s))
            body["consolidations"].append(c)
    def secret(t):   # (signers, root, setter) over registry keys, or (None, root, setter, sk) for an outside key
        return t[3] if t[0] is None else sum(sks[v] for v in t[0]) % CURVE_ORDER or 1
    sk_bytes = b"".join(secret(t).to_bytes(32, "big") for t in todo)
    sigs = sign_fn(sk_bytes, b"".join(t[1] for t in todo))
    for k, t in enumerate(todo):
        t[2](sigs[96 * k:96 * k + 96])
    msg = S.serialize(S.BEACON_BLOCK_BY_FORK[fork], block)
    root = block_root_fn(msg)
    sig = sign_fn(sks[proposer].to_bytes(32, "big"), _sha(root + domain(DOMAIN_PROPOSER, epoch)))
    return struct.pack("<I", 100) + sig + msg, root
