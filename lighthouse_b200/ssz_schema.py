"""Minimal SSZ type descriptors + serializer for the Deneb BeaconBlock (mainnet preset), used to BUILD synthetic
blocks (consensus/types/src/beacon_block.rs:56-78, beacon_block_body.rs:70-121, execution_payload.rs:54-95 and the
operation containers).  Serialization only — hashing is the CUDA library's job (tests/ssz_spec.py holds the
from-spec hashlib hash_tree_root used to pin the oracle).

Types:  ("uint", nbytes) | ("bytes", n) fixed byte vector | ("bytelist", limit) | ("bitlist", limit) |
        ("bitvector", nbits) | ("vector", elem, n) | ("list", elem, limit) | ("container", [(name, type), ...])
Values: int | bytes | list[bool] for bit types | list | dict.
"""

U64 = ("uint", 8)
U256 = ("uint", 32)
B20, B32, B48, B96 = ("bytes", 20), ("bytes", 32), ("bytes", 48), ("bytes", 96)


def C(*fields):
    return ("container", list(fields))


Checkpoint = C(("epoch", U64), ("root", B32))
AttestationData = C(("slot", U64), ("index", U64), ("beacon_block_root", B32), ("source", Checkpoint),
                    ("target", Checkpoint))
BeaconBlockHeader = C(("slot", U64), ("proposer_index", U64), ("parent_root", B32), ("state_root", B32),
                      ("body_root", B32))
SignedBeaconBlockHeader = C(("message", BeaconBlockHeader), ("signature", B96))
ProposerSlashing = C(("signed_header_1", SignedBeaconBlockHeader), ("signed_header_2", SignedBeaconBlockHeader))
IndexedAttestation = C(("attesting_indices", ("list", U64, 2048)), ("data", AttestationData), ("signature", B96))
AttesterSlashing = C(("attestation_1", IndexedAttestation), ("attestation_2", IndexedAttestation))
Attestation = C(("aggregation_bits", ("bitlist", 2048)), ("data", AttestationData), ("signature", B96))
Eth1Data = C(("deposit_root", B32), ("deposit_count", U64), ("block_hash", B32))
DepositData = C(("pubkey", B48), ("withdrawal_credentials", B32), ("amount", U64), ("signature", B96))
Deposit = C(("proof", ("vector", B32, 33)), ("data", DepositData))
VoluntaryExit = C(("epoch", U64), ("validator_index", U64))
SignedVoluntaryExit = C(("message", VoluntaryExit), ("signature", B96))
SyncAggregate = C(("sync_committee_bits", ("bitvector", 512)), ("sync_committee_signature", B96))
Withdrawal = C(("index", U64), ("validator_index", U64), ("address", B20), ("amount", U64))
BlsToExecutionChange = C(("validator_index", U64), ("from_bls_pubkey", B48), ("to_execution_address", B20))
SignedBlsToExecutionChange = C(("message", BlsToExecutionChange), ("signature", B96))
ExecutionPayloadDeneb = C(
    ("parent_hash", B32), ("fee_recipient", B20), ("state_root", B32), ("receipts_root", B32),
    ("logs_bloom", ("bytes", 256)), ("prev_randao", B32), ("block_number", U64), ("gas_limit", U64),
    ("gas_used", U64), ("timestamp", U64), ("extra_data", ("bytelist", 32)), ("base_fee_per_gas", U256),
    ("block_hash", B32), ("transactions", ("list", ("bytelist", 1 << 30), 1 << 20)),
    ("withdrawals", ("list", Withdrawal, 16)), ("blob_gas_used", U64), ("excess_blob_gas", U64))
BeaconBlockBodyDeneb = C(
    ("randao_reveal", B96), ("eth1_data", Eth1Data), ("graffiti", B32),
    ("proposer_slashings", ("list", ProposerSlashing, 16)), ("attester_slashings", ("list", AttesterSlashing, 2)),
    ("attestations", ("list", Attestation, 128)), ("deposits", ("list", Deposit, 16)),
    ("voluntary_exits", ("list", SignedVoluntaryExit, 16)), ("sync_aggregate", SyncAggregate),
    ("execution_payload", ExecutionPayloadDeneb),
    ("bls_to_execution_changes", ("list", SignedBlsToExecutionChange, 16)),
    ("blob_kzg_commitments", ("list", B48, 4096)))
BeaconBlockDeneb = C(("slot", U64), ("proposer_index", U64), ("parent_root", B32), ("state_root", B32),
                     ("body", BeaconBlockBodyDeneb))
SignedBeaconBlockDeneb = C(("message", BeaconBlockDeneb), ("signature", B96))


def is_fixed(t):
    k = t[0]
    if k in ("uint", "bytes", "bitvector"):
        return True
    if k in ("bytelist", "bitlist", "list"):
        return False
    if k == "vector":
        return is_fixed(t[1])
    return all(is_fixed(ft) for _, ft in t[1])


def fixed_size(t):
    k = t[0]
    if k in ("uint", "bytes"):
        return t[1]
    if k == "bitvector":
        return (t[1] + 7) // 8
    if k == "vector":
        return t[2] * fixed_size(t[1])
    return sum(fixed_size(ft) if is_fixed(ft) else 4 for _, ft in t[1])


def pack_bits(bits, delimiter):
    bits = list(bits) + ([True] if delimiter else [])
    out = bytearray((len(bits) + 7) // 8)
    for i, b in enumerate(bits):
        if b:
            out[i // 8] |= 1 << (i % 8)
    return bytes(out)


def _sequence(parts, fixed_flags):
    """SSZ layout of a heterogeneous sequence: fixed parts inline, variable parts behind 4-byte offsets."""
    head = sum(len(p) if f else 4 for p, f in zip(parts, fixed_flags))
    out, tail = bytearray(), bytearray()
    for p, f in zip(parts, fixed_flags):
        if f:
            out += p
        else:
            out += (head + len(tail)).to_bytes(4, "little")
            tail += p
    return bytes(out + tail)


def serialize(t, v):
    k = t[0]
    if k == "uint":
        return int(v).to_bytes(t[1], "little")
    if k == "bytes":
        assert len(v) == t[1], (t, len(v))
        return bytes(v)
    if k == "bytelist":
        assert len(v) <= t[1]
        return bytes(v)
    if k == "bitlist":
        assert len(v) <= t[1]
        return pack_bits(v, True)
    if k == "bitvector":
        assert len(v) == t[1]
        return pack_bits(v, False)
    if k in ("vector", "list"):
        if k == "vector":
            assert len(v) == t[2]
        else:
            assert len(v) <= t[2]
        parts = [serialize(t[1], e) for e in v]
        return _sequence(parts, [is_fixed(t[1])] * len(parts))
    parts = [serialize(ft, v[name]) for name, ft in t[1]]
    return _sequence(parts, [is_fixed(ft) for _, ft in t[1]])


# ---- BeaconStateDeneb (consensus/types/src/beacon_state.rs:339-490, mainnet sizes eth_spec.rs:389-430) ----------
B4 = ("bytes", 4)
Fork = C(("previous_version", B4), ("current_version", B4), ("epoch", U64))
Validator = C(("pubkey", B48), ("withdrawal_credentials", B32), ("effective_balance", U64), ("slashed", ("uint", 1)),
              ("activation_eligibility_epoch", U64), ("activation_epoch", U64), ("exit_epoch", U64),
              ("withdrawable_epoch", U64))
SyncCommittee = C(("pubkeys", ("vector", B48, 512)), ("aggregate_pubkey", B48))
ExecutionPayloadHeaderDeneb = C(
    ("parent_hash", B32), ("fee_recipient", B20), ("state_root", B32), ("receipts_root", B32),
    ("logs_bloom", ("bytes", 256)), ("prev_randao", B32), ("block_number", U64), ("gas_limit", U64),
    ("gas_used", U64), ("timestamp", U64), ("extra_data", ("bytelist", 32)), ("base_fee_per_gas", U256),
    ("block_hash", B32), ("transactions_root", B32), ("withdrawals_root", B32), ("blob_gas_used", U64),
    ("excess_blob_gas", U64))
HistoricalSummary = C(("block_summary_root", B32), ("state_summary_root", B32))
BeaconStateDeneb = C(
    ("genesis_time", U64), ("genesis_validators_root", B32), ("slot", U64), ("fork", Fork),
    ("latest_block_header", BeaconBlockHeader), ("block_roots", ("vector", B32, 8192)),
    ("state_roots", ("vector", B32, 8192)), ("historical_roots", ("list", B32, 1 << 24)), ("eth1_data", Eth1Data),
    ("eth1_data_votes", ("list", Eth1Data, 2048)), ("eth1_deposit_index", U64),
    ("validators", ("list", Validator, 1 << 40)), ("balances", ("list", U64, 1 << 40)),
    ("randao_mixes", ("vector", B32, 65536)), ("slashings", ("vector", U64, 8192)),
    ("previous_epoch_participation", ("list", ("uint", 1), 1 << 40)),
    ("current_epoch_participation", ("list", ("uint", 1), 1 << 40)), ("justification_bits", ("bitvector", 4)),
    ("previous_justified_checkpoint", Checkpoint), ("current_justified_checkpoint", Checkpoint),
    ("finalized_checkpoint", Checkpoint), ("inactivity_scores", ("list", U64, 1 << 40)),
    ("current_sync_committee", SyncCommittee), ("next_sync_committee", SyncCommittee),
    ("latest_execution_payload_header", ExecutionPayloadHeaderDeneb), ("next_withdrawal_index", U64),
    ("next_withdrawal_validator_index", U64), ("historical_summaries", ("list", HistoricalSummary, 1 << 24)))


# ---- the earlier post-Altair variants of the superstruct (beacon_state.rs:224-571): prefixes of the Deneb field list
# with narrower execution payload headers
ExecutionPayloadHeaderBellatrix = C(*ExecutionPayloadHeaderDeneb[1][:14])
ExecutionPayloadHeaderCapella = C(*ExecutionPayloadHeaderDeneb[1][:15])
_f = BeaconStateDeneb[1]
BeaconStateAltair = C(*_f[:24])
BeaconStateBellatrix = C(*(_f[:24] + [("latest_execution_payload_header", ExecutionPayloadHeaderBellatrix)]))
BeaconStateCapella = C(*(_f[:24] + [("latest_execution_payload_header", ExecutionPayloadHeaderCapella)] + _f[25:]))
# ---- Electra as in this revision of the reference (beacon_state.rs:487-525, execution_payload_header.rs:88-93,
# pending_balance_deposit.rs:21, pending_partial_withdrawal.rs:22, pending_consolidation.rs:21; limits eth_spec.rs:433-435)
ExecutionPayloadHeaderElectra = C(*(ExecutionPayloadHeaderDeneb[1] + [("deposit_requests_root", B32),
                                                                     ("withdrawal_requests_root", B32)]))
PendingBalanceDeposit = C(("index", U64), ("amount", U64))
PendingPartialWithdrawal = C(("index", U64), ("amount", U64), ("withdrawable_epoch", U64))
PendingConsolidation = C(("source_index", U64), ("target_index", U64))
BeaconStateElectra = C(*(_f[:24] + [("latest_execution_payload_header", ExecutionPayloadHeaderElectra)] + _f[25:] + [
    ("deposit_requests_start_index", U64), ("deposit_balance_to_consume", U64), ("exit_balance_to_consume", U64),
    ("earliest_exit_epoch", U64), ("consolidation_balance_to_consume", U64), ("earliest_consolidation_epoch", U64),
    ("pending_balance_deposits", ("list", PendingBalanceDeposit, 1 << 27)),
    ("pending_partial_withdrawals", ("list", PendingPartialWithdrawal, 1 << 27)),
    ("pending_consolidations", ("list", PendingConsolidation, 1 << 18))]))
# ---- Base (phase0: beacon_state.rs:225-406 Base fields, pending_attestation.rs:25-32; limits eth_spec.rs:389-430):
# Altair's first 21 fields with the participation lists replaced by pending-attestation lists
PendingAttestation = C(("aggregation_bits", ("bitlist", 2048)), ("data", AttestationData), ("inclusion_delay", U64),
                       ("proposer_index", U64))
BeaconStateBase = C(*(_f[:15] + [("previous_epoch_attestations", ("list", PendingAttestation, 4096)),
                                 ("current_epoch_attestations", ("list", PendingAttestation, 4096))] + _f[17:21]))
BEACON_STATE_BY_FORK = {"base": BeaconStateBase, "altair": BeaconStateAltair, "bellatrix": BeaconStateBellatrix, "capella": BeaconStateCapella,
                        "deneb": BeaconStateDeneb, "electra": BeaconStateElectra}


# ---- the earlier variants of the BeaconBlock superstruct (beacon_block.rs:41-90, beacon_block_body.rs:43-110)
def _block_of(body):
    return C(("slot", U64), ("proposer_index", U64), ("parent_root", B32), ("state_root", B32), ("body", body))


_pf, _bf = ExecutionPayloadDeneb[1], BeaconBlockBodyDeneb[1]
ExecutionPayloadBellatrix = C(*_pf[:14])
ExecutionPayloadCapella = C(*_pf[:15])
BeaconBlockBodyBase = C(*_bf[:8])   # beacon_block_body.rs:33-119: no sync_aggregate
BeaconBlockBodyAltair = C(*_bf[:9])
BeaconBlockBodyBellatrix = C(*(_bf[:9] + [("execution_payload", ExecutionPayloadBellatrix)]))
BeaconBlockBodyCapella = C(*(_bf[:9] + [("execution_payload", ExecutionPayloadCapella)] + _bf[10:11]))
# ---- Electra as in this revision of the reference (beacon_block_body.rs:70-121, attestation.rs:76-82,
# indexed_attestation.rs:57-62, execution_payload.rs:54-101, deposit_request.rs:23-29,
# execution_layer_withdrawal_request.rs:23-26, signed_consolidation.rs:23-24, consolidation.rs:24-27; limits
# eth_spec.rs:395-440: MaxValidatorsPerSlot 131072, MaxCommitteesPerSlot 64)
IndexedAttestationElectra = C(("attesting_indices", ("list", U64, 131072)), ("data", AttestationData), ("signature", B96))
AttesterSlashingElectra = C(("attestation_1", IndexedAttestationElectra), ("attestation_2", IndexedAttestationElectra))
AttestationElectra = C(("aggregation_bits", ("bitlist", 131072)), ("data", AttestationData),
                       ("committee_bits", ("bitvector", 64)), ("signature", B96))
DepositRequest = C(("pubkey", B48), ("withdrawal_credentials", B32), ("amount", U64), ("signature", B96), ("index", U64))
ExecutionLayerWithdrawalRequest = C(("source_address", B20), ("validator_pubkey", B48), ("amount", U64))
Consolidation = C(("source_index", U64), ("target_index", U64), ("epoch", U64))
SignedConsolidation = C(("message", Consolidation), ("signature", B96))
ExecutionPayloadElectra = C(*(_pf + [("deposit_requests", ("list", DepositRequest, 8192)),
                                     ("withdrawal_requests", ("list", ExecutionLayerWithdrawalRequest, 16))]))
_electra_body = {"attester_slashings": ("list", AttesterSlashingElectra, 1), "attestations": ("list", AttestationElectra, 8),
                 "execution_payload": ExecutionPayloadElectra}
BeaconBlockBodyElectra = C(*([(n, _electra_body.get(n, t)) for n, t in _bf] +
                             [("consolidations", ("list", SignedConsolidation, 1))]))
BEACON_BLOCK_BODY_BY_FORK = {"base": BeaconBlockBodyBase, "altair": BeaconBlockBodyAltair, "bellatrix": BeaconBlockBodyBellatrix,
                             "capella": BeaconBlockBodyCapella, "deneb": BeaconBlockBodyDeneb,
                             "electra": BeaconBlockBodyElectra}
BEACON_BLOCK_BY_FORK = {k: _block_of(v) for k, v in BEACON_BLOCK_BODY_BY_FORK.items()}
BeaconBlockBase = BEACON_BLOCK_BY_FORK["base"]
EXECUTION_PAYLOAD_BY_FORK = {"bellatrix": ExecutionPayloadBellatrix, "capella": ExecutionPayloadCapella,
                             "deneb": ExecutionPayloadDeneb, "electra": ExecutionPayloadElectra}
EXECUTION_PAYLOAD_HEADER_BY_FORK = {"bellatrix": ExecutionPayloadHeaderBellatrix, "capella": ExecutionPayloadHeaderCapella,
                                    "deneb": ExecutionPayloadHeaderDeneb, "electra": ExecutionPayloadHeaderElectra}
BLINDED_BEACON_BLOCK_BODY_BY_FORK = {
    f: C(*[(n, EXECUTION_PAYLOAD_HEADER_BY_FORK[f]) if n == "execution_payload" else (n, t) for n, t in b[1]])
    for f, b in BEACON_BLOCK_BODY_BY_FORK.items() if f not in ("base", "altair")}
BLINDED_BEACON_BLOCK_BY_FORK = {k: _block_of(v) for k, v in BLINDED_BEACON_BLOCK_BODY_BY_FORK.items()}

# BlindedBeaconBlock (beacon_block.rs:80; payload.rs BlindedPayload): the body carries the payload HEADER
BlindedBeaconBlockBodyDeneb = C(*[(n, ExecutionPayloadHeaderDeneb) if n == "execution_payload" else (n, t)
                                 for n, t in BeaconBlockBodyDeneb[1]])
BlindedBeaconBlockDeneb = C(("slot", U64), ("proposer_index", U64), ("parent_root", B32), ("state_root", B32),
                            ("body", BlindedBeaconBlockBodyDeneb))
