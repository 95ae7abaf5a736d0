#!/usr/bin/env python3
"""Extract the reference's own in-tree golden vectors into tests/golden/ (run in the build container only;
/root/reference does not exist on the GPU box).  Sources (all under /root/reference):
  common/eth2_network_config/built_in_network_configs/{mainnet,sepolia,gnosis}/genesis.ssz.zip
      phase0 genesis BeaconState; bytes 8..40 = genesis_validators_root = hash_tree_root(validators)
      (checked by common/eth2_network_config/src/lib.rs:227-233); mainnet and Sepolia also whole, as the bytes
      around the validators list, with their state roots (and mainnet's genesis block root)
  validator_manager/test_vectors/vectors/*/validator_keys/deposit_data-*.json
      22 (pubkey, signature, deposit_message_root, deposit_data_root) entries, asserted valid by
      validator_manager/src/create_validators.rs:749-768
  common/eth2_interop_keypairs/specs/keygen_10_validators.yaml  (sk -> pk, tests/generation.rs:6-64)
"""
import glob, io, json, lzma, os, struct, sys, zipfile
import yaml

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
os.makedirs(OUT, exist_ok=True)

# phase0 BeaconState fixed part: offset of the `validators` u32 offset (SURVEY §8c)
VAL_OFF_POS = 8 + 32 + 8 + 16 + 112 + 2 * 8192 * 32 + 4 + 72 + 4 + 8
meta = {}
for net in ("mainnet", "sepolia", "gnosis"):
    z = zipfile.ZipFile(f"{REF}/common/eth2_network_config/built_in_network_configs/{net}/genesis.ssz.zip")
    state = z.read(z.namelist()[0])
    o_val, o_bal = struct.unpack_from("<II", state, VAL_OFF_POS)
    vals = state[o_val:o_bal]
    assert len(vals) % 121 == 0
    with lzma.open(os.path.join(OUT, f"genesis_validators_{net}.bin.xz"), "wb", preset=9) as f:
        f.write(vals)
    meta[net] = {"n_validators": len(vals) // 121, "genesis_validators_root": state[8:40].hex()}
json.dump(meta, open(os.path.join(OUT, "genesis_validators.json"), "w"), indent=1)

# The rest of the mainnet and Sepolia genesis states (complete phase0 BeaconStates): the bytes before and after the
# validators list, which tests put back together with genesis_validators_{net}.bin.xz.  Their roots come from the
# from-spec merkleization in tests/ssz_spec.py; the mainnet ones equal mainnet's published genesis state and block
# roots, which pins that merkleizer for phase0 states.  Gnosis is left out: it uses the Gnosis preset (2048 pending
# attestations, 1024 eth1 votes), and its mainnet-preset root is not its genesis root.
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from lighthouse_b200 import ssz_schema as S  # noqa: E402
from tests.ssz_spec import deserialize, hash_tree_root  # noqa: E402

PUBLISHED = {"mainnet": ("7e76880eb67bbdc86250aa578958e9d0675e64e714337855204fb5abaaf82c2b",
                         "4d611d5b93fdab69013a7f0a2f961caca0c853f87cfe9595fe50038163079360")}
states = {}
for net in ("mainnet", "sepolia"):
    z = zipfile.ZipFile(f"{REF}/common/eth2_network_config/built_in_network_configs/{net}/genesis.ssz.zip")
    state = z.read(z.namelist()[0])
    o_val, o_bal = struct.unpack_from("<II", state, VAL_OFF_POS)
    with lzma.open(os.path.join(OUT, f"genesis_state_rest_{net}.bin.xz"), "wb", preset=9) as f:
        f.write(state[:o_val] + state[o_bal:])
    v = deserialize(S.BeaconStateBase, state)
    root = hash_tree_root(S.BeaconStateBase, v)
    empty_body = {"randao_reveal": bytes(96), "eth1_data": {"deposit_root": bytes(32), "deposit_count": 0,
                                                            "block_hash": bytes(32)}, "graffiti": bytes(32),
                  "proposer_slashings": [], "attester_slashings": [], "attestations": [], "deposits": [],
                  "voluntary_exits": []}
    block = {"slot": 0, "proposer_index": 0, "parent_root": bytes(32), "state_root": root, "body": empty_body}
    block_root = hash_tree_root(S.BeaconBlockBase, block)
    src = f"common/eth2_network_config/built_in_network_configs/{net}/genesis.ssz.zip"
    e = {"source": src, "ssz_bytes": len(state), "validators_offset": o_val, "validators_end": o_bal,
         "n_validators": (o_bal - o_val) // 121, "state_root": root.hex(),
         "state_root_provenance": "hash_tree_root(BeaconStateBase) by tests/ssz_spec.py over the SSZ in " + src}
    if net in PUBLISHED:
        assert (root.hex(), block_root.hex()) == PUBLISHED[net], (net, root.hex(), block_root.hex())
        e["state_root_provenance"] += "; equals mainnet's published genesis state root"
        e["genesis_block_root"] = block_root.hex()
        e["genesis_block_root_provenance"] = ("hash_tree_root(BeaconBlockBase{slot 0, proposer_index 0, parent_root 0, "
                                              "state_root, empty body}) by tests/ssz_spec.py; equals mainnet's "
                                              "published genesis block root")
    states[net] = e
json.dump(states, open(os.path.join(OUT, "genesis_states.json"), "w"), indent=1)

deps = []
for p in sorted(glob.glob(f"{REF}/validator_manager/test_vectors/vectors/*/validator_keys/deposit_data-*.json")):
    for d in json.load(open(p)):
        deps.append({k: d[k] for k in ("pubkey", "withdrawal_credentials", "amount", "signature",
                                        "deposit_message_root", "deposit_data_root", "fork_version")}
                    | {"source": os.path.relpath(p, REF)})
json.dump(deps, open(os.path.join(OUT, "deposit_data.json"), "w"), indent=1)

kp = yaml.safe_load(open(f"{REF}/common/eth2_interop_keypairs/specs/keygen_10_validators.yaml"))
json.dump(kp, open(os.path.join(OUT, "interop_keypairs.json"), "w"), indent=1)
print({k: v["n_validators"] for k, v in meta.items()}, len(deps), "deposits", len(kp), "keypairs")
