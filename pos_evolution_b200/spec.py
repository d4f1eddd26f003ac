"""pyspec-signature host layer over the H100 engine.

Keeps the names, argument meaning and error behaviour (AssertionError = invalid) of the functions
quoted in pos-evolution.md, line numbers cited per function, so that it can stand
in for the executable consensus spec on the path
    process_attestation (:722) -> is_valid_indexed_attestation -> bls.FastAggregateVerify
    on_attestation (:963/:1423) -> update_latest_messages (:1435) -> get_head (:1102).
Python here only marshals: committee shuffling (SHA-256 via hashlib, vectorised numpy -- the GPU
version is SURVEY.md section 8(f)-1), SSZ signing roots, participation-flag bookkeeping.  Signature
aggregation/verification and the fork-choice weights/head run on the GPU through engine.Engine.
This module never imports oracle/.
"""
import hashlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Set

import numpy as np

from .engine import Engine

FAR_FUTURE_EPOCH = 2**64 - 1
GENESIS_EPOCH = 0
ZERO32 = bytes(32)
G2_POINT_AT_INFINITY = bytes([0xC0]) + bytes(95)
DOMAIN_BEACON_PROPOSER = bytes.fromhex("00000000")
DOMAIN_BEACON_ATTESTER = bytes.fromhex("01000000")
DOMAIN_SELECTION_PROOF = bytes.fromhex("05000000")             # upstream phase 0 validator spec
DOMAIN_AGGREGATE_AND_PROOF = bytes.fromhex("06000000")
DOMAIN_SYNC_COMMITTEE = bytes.fromhex("07000000")
DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF = bytes.fromhex("08000000")     # upstream Altair
DOMAIN_CONTRIBUTION_AND_PROOF = bytes.fromhex("09000000")
SYNC_REWARD_WEIGHT = 2
TIMELY_SOURCE_FLAG_INDEX, TIMELY_TARGET_FLAG_INDEX, TIMELY_HEAD_FLAG_INDEX = 0, 1, 2
PARTICIPATION_FLAG_WEIGHTS = [14, 26, 14]
PROPOSER_WEIGHT = 8
WEIGHT_DENOMINATOR = 64
BASE_REWARD_FACTOR = 64
JUSTIFICATION_BITS_LENGTH = 4


@dataclass(frozen=True)
class Preset:
    name: str
    SLOTS_PER_EPOCH: int
    MAX_COMMITTEES_PER_SLOT: int
    TARGET_COMMITTEE_SIZE: int
    SHUFFLE_ROUND_COUNT: int
    EPOCHS_PER_HISTORICAL_VECTOR: int
    SLOTS_PER_HISTORICAL_ROOT: int
    MAX_VALIDATORS_PER_COMMITTEE: int = 2048
    MIN_ATTESTATION_INCLUSION_DELAY: int = 1
    MIN_SEED_LOOKAHEAD: int = 1
    MAX_EFFECTIVE_BALANCE: int = 32 * 10**9
    EFFECTIVE_BALANCE_INCREMENT: int = 10**9
    PROPOSER_SCORE_BOOST: int = 40
    SYNC_COMMITTEE_SIZE: int = 512
    EPOCHS_PER_SYNC_COMMITTEE_PERIOD: int = 256
    MAX_ATTESTATIONS: int = 128                   # BeaconBlockBody.attestations limit (:639)
    VALIDATOR_REGISTRY_LIMIT: int = 2**40         # list limits and vector lengths of BeaconState (:338-374)
    HISTORICAL_ROOTS_LIMIT: int = 2**24
    EPOCHS_PER_SLASHINGS_VECTOR: int = 8192
    EPOCHS_PER_ETH1_VOTING_PERIOD: int = 64
    TARGET_AGGREGATORS_PER_COMMITTEE: int = 16    # upstream phase 0 validator spec (is_aggregator)
    ATTESTATION_PROPAGATION_SLOT_RANGE: int = 32  # upstream phase 0 p2p spec (beacon_aggregate_and_proof)
    SYNC_COMMITTEE_SUBNET_COUNT: int = 4          # upstream Altair validator spec (sync_committee_{subnet_id})
    TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE: int = 16      # upstream Altair validator spec (is_sync_committee_aggregator)


MAINNET = Preset("mainnet", 32, 64, 128, 90, 65536, 8192)
MINIMAL = Preset("minimal", 8, 4, 4, 10, 64, 64, SYNC_COMMITTEE_SIZE=32, EPOCHS_PER_SYNC_COMMITTEE_PERIOD=8, EPOCHS_PER_SLASHINGS_VECTOR=64,
                 EPOCHS_PER_ETH1_VOTING_PERIOD=4)


# ----------------------------------------------------------------------------- containers
@dataclass
class Validator:                       # pos-evolution.md:36-45
    pubkey: bytes
    effective_balance: int
    slashed: bool = False
    activation_epoch: int = 0
    exit_epoch: int = FAR_FUTURE_EPOCH
    withdrawal_credentials: bytes = ZERO32
    activation_eligibility_epoch: int = 0
    withdrawable_epoch: int = FAR_FUTURE_EPOCH


@dataclass(frozen=True)
class Checkpoint:                      # :219-221
    epoch: int = 0
    root: bytes = ZERO32


@dataclass(frozen=True)
class AttestationData:                 # :689-697
    slot: int
    index: int
    beacon_block_root: bytes
    source: Checkpoint
    target: Checkpoint


@dataclass
class Attestation:                     # :714-717
    aggregation_bits: List[bool]
    data: AttestationData
    signature: bytes


@dataclass
class ElectraAttestation:              # upstream Electra beacon-chain.md (EIP-7549); SSZ field order as written
    aggregation_bits: List[bool]       # the bit rows of the committees committee_bits names, back to back
    data: AttestationData              # data.index == 0
    signature: bytes
    committee_bits: List[bool]         # Bitvector[MAX_COMMITTEES_PER_SLOT]


@dataclass
class SingleAttestation:               # upstream Electra beacon-chain.md (EIP-7549); the beacon_attestation_{subnet_id} gossip message
    committee_index: int
    attester_index: int
    data: AttestationData              # data.index == 0
    signature: bytes


@dataclass
class BlockAttestations:               # the attestations of one block (BeaconBlockBody.attestations, :639) and what processing them needs
    slot: int                          # the block's slot: state.slot when process_block runs
    proposer_index: int                # the block's proposer, credited with the proposer rewards (:753-754)
    root: bytes                        # the block's root: state.block_roots of its slot and of the slots skipped after it
    attestations: List[Attestation]


@dataclass
class AggregateAndProof:               # upstream phase 0 validator spec
    aggregator_index: int
    aggregate: Attestation
    selection_proof: bytes


@dataclass
class SignedAggregateAndProof:         # upstream phase 0 validator spec; the beacon_aggregate_and_proof gossip message
    message: AggregateAndProof
    signature: bytes


@dataclass
class IndexedAttestation:
    attesting_indices: List[int]
    data: AttestationData
    signature: bytes


@dataclass
class AttesterSlashing:                # pos-evolution.md:1160-1162
    attestation_1: "IndexedAttestation"
    attestation_2: "IndexedAttestation"


@dataclass(frozen=True)
class LatestMessage:                   # :287-289
    epoch: int
    root: bytes


@dataclass
class Fork:
    previous_version: bytes = bytes(4)
    current_version: bytes = bytes(4)
    epoch: int = 0


@dataclass
class BeaconBlock:                     # :671-676 (fields fork choice reads)
    slot: int
    parent_root: bytes


@dataclass
class SyncCommittee:                   # BeaconState.current_sync_committee / next_sync_committee (:371-372); Altair container
    pubkeys: List[bytes]               # SYNC_COMMITTEE_SIZE keys; a validator may appear more than once
    aggregate_pubkey: bytes


@dataclass
class SyncAggregate:                   # Altair BeaconBlockBody.sync_aggregate
    sync_committee_bits: List[bool]    # Bitvector[SYNC_COMMITTEE_SIZE]
    sync_committee_signature: bytes


@dataclass
class SyncCommitteeMessage:            # pos-evolution.md:548-557; the sync_committee_{subnet_id} gossip message
    slot: int
    beacon_block_root: bytes
    validator_index: int
    signature: bytes


@dataclass
class SyncCommitteeContribution:       # upstream Altair validator spec
    slot: int
    beacon_block_root: bytes
    subcommittee_index: int
    aggregation_bits: List[bool]       # Bitvector[SYNC_COMMITTEE_SIZE // SYNC_COMMITTEE_SUBNET_COUNT]
    signature: bytes


@dataclass
class SyncAggregatorSelectionData:     # upstream Altair validator spec: what a selection proof signs
    slot: int
    subcommittee_index: int


@dataclass
class ContributionAndProof:            # upstream Altair validator spec
    aggregator_index: int
    contribution: SyncCommitteeContribution
    selection_proof: bytes


@dataclass
class SignedContributionAndProof:      # upstream Altair validator spec; the sync_committee_contribution_and_proof gossip message
    message: ContributionAndProof
    signature: bytes


class SyncAggregates(dict):
    """{beacon_block_root: SyncAggregate} of Spec.validate_sync_committee_messages; a root nobody signed gives the empty aggregate (no bits,
    the G2 infinity signature), which eth_fast_aggregate_verify accepts"""

    def __init__(self, size, *args):
        super().__init__(*args)
        self.size = size

    def __missing__(self, root):
        return SyncAggregate([False] * self.size, G2_POINT_AT_INFINITY)


@dataclass
class BeaconBlockHeader:               # named in BeaconState (:343); fields as in upstream phase 0
    slot: int = 0
    proposer_index: int = 0
    parent_root: bytes = ZERO32
    state_root: bytes = ZERO32
    body_root: bytes = ZERO32


@dataclass
class Eth1Data:                        # named in BeaconState (:348-349); fields as in upstream phase 0
    deposit_root: bytes = ZERO32
    deposit_count: int = 0
    block_hash: bytes = ZERO32


@dataclass
class ExecutionPayloadHeader:          # named in BeaconState (:374); fields as in upstream Bellatrix
    parent_hash: bytes = ZERO32
    fee_recipient: bytes = bytes(20)
    state_root: bytes = ZERO32
    receipts_root: bytes = ZERO32
    logs_bloom: bytes = bytes(256)
    prev_randao: bytes = ZERO32
    block_number: int = 0
    gas_limit: int = 0
    gas_used: int = 0
    timestamp: int = 0
    extra_data: bytes = b""            # ByteList[32]
    base_fee_per_gas: int = 0          # uint256
    block_hash: bytes = ZERO32
    transactions_root: bytes = ZERO32


@dataclass
class BeaconState:                     # :338-374; the fields after next_sync_committee only enter hash_tree_root_state
    slot: int
    fork: Fork
    genesis_validators_root: bytes
    validators: List[Validator]
    balances: List[int]
    randao_mixes: List[bytes]
    block_roots: List[bytes]
    previous_epoch_participation: List[int]
    current_epoch_participation: List[int]
    previous_justified_checkpoint: Checkpoint = Checkpoint()
    current_justified_checkpoint: Checkpoint = Checkpoint()
    finalized_checkpoint: Checkpoint = Checkpoint()
    justification_bits: List[int] = field(default_factory=lambda: [0] * JUSTIFICATION_BITS_LENGTH)
    current_sync_committee: Optional[SyncCommittee] = None          # :371
    next_sync_committee: Optional[SyncCommittee] = None             # :372
    genesis_time: int = 0
    latest_block_header: BeaconBlockHeader = field(default_factory=BeaconBlockHeader)
    state_roots: Optional[List[bytes]] = None                        # Vector[Root, SLOTS_PER_HISTORICAL_ROOT]; None = all zero
    historical_roots: List[bytes] = field(default_factory=list)
    eth1_data: Eth1Data = field(default_factory=Eth1Data)
    eth1_data_votes: List[Eth1Data] = field(default_factory=list)
    eth1_deposit_index: int = 0
    slashings: Optional[List[int]] = None                            # Vector[Gwei, EPOCHS_PER_SLASHINGS_VECTOR]; None = all zero
    inactivity_scores: List[int] = field(default_factory=list)
    latest_execution_payload_header: ExecutionPayloadHeader = field(default_factory=ExecutionPayloadHeader)


@dataclass
class Store:                           # :890-901
    time: int
    genesis_time: int
    justified_checkpoint: Checkpoint
    finalized_checkpoint: Checkpoint
    best_justified_checkpoint: Checkpoint
    proposer_boost_root: bytes
    equivocating_indices: Set[int]
    blocks: Dict[bytes, BeaconBlock] = field(default_factory=dict)
    block_states: Dict[bytes, BeaconState] = field(default_factory=dict)
    checkpoint_states: Dict[Checkpoint, BeaconState] = field(default_factory=dict)
    latest_messages: Dict[int, LatestMessage] = field(default_factory=dict)


# ----------------------------------------------------------------------------- SSZ-lite
def sha256(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()


def _u64_chunk(v: int) -> bytes:
    return int(v).to_bytes(8, "little") + bytes(24)


def _merkle(chunks):
    n = 1
    while n < len(chunks):
        n *= 2
    layer = list(chunks) + [ZERO32] * (n - len(chunks))
    while len(layer) > 1:
        layer = [sha256(layer[i] + layer[i + 1]) for i in range(0, len(layer), 2)]
    return layer[0]


def hash_tree_root_checkpoint(c: Checkpoint) -> bytes:
    return _merkle([_u64_chunk(c.epoch), bytes(c.root)])


def hash_tree_root_attestation_data(d: AttestationData) -> bytes:
    return _merkle([_u64_chunk(d.slot), _u64_chunk(d.index), bytes(d.beacon_block_root),
                    hash_tree_root_checkpoint(d.source), hash_tree_root_checkpoint(d.target)])


def serialize_attestation_data(d: AttestationData) -> bytes:
    """SSZ serialisation of the fixed-size container (128 bytes): the record format of Engine.signing_roots."""
    return (int(d.slot).to_bytes(8, "little") + int(d.index).to_bytes(8, "little") + bytes(d.beacon_block_root)
            + int(d.source.epoch).to_bytes(8, "little") + bytes(d.source.root) + int(d.target.epoch).to_bytes(8, "little") + bytes(d.target.root))


def deserialize_attestation_data(b: bytes) -> AttestationData:
    u = lambda o: int.from_bytes(b[o:o + 8], "little")       # noqa: E731
    return AttestationData(slot=u(0), index=u(8), beacon_block_root=bytes(b[16:48]), source=Checkpoint(u(48), bytes(b[56:88])),
                           target=Checkpoint(u(88), bytes(b[96:128])))


def serialize_attestation(att: Attestation) -> bytes:
    """SSZ wire form (:714-717): [offset of aggregation_bits = 228][data][signature][Bitlist with its delimiter bit]."""
    n = len(att.aggregation_bits)
    bl = bytearray(pack_bits([list(att.aggregation_bits)], stride=n // 8 + 1)[0].tobytes())
    bl[n >> 3] |= 1 << (n & 7)
    return (228).to_bytes(4, "little") + serialize_attestation_data(att.data) + bytes(att.signature) + bytes(bl)


def serialize_attestation_electra(att: ElectraAttestation) -> bytes:
    """SSZ wire form: [offset of aggregation_bits = 228 + ceil(M / 8)][data][signature][committee_bits Bitvector[M]][Bitlist with its
    delimiter bit], M = len(committee_bits)."""
    M, n = len(att.committee_bits), len(att.aggregation_bits)
    cb = pack_bits([list(att.committee_bits)], stride=(M + 7) // 8)[0].tobytes()
    bl = bytearray(pack_bits([list(att.aggregation_bits)], stride=n // 8 + 1)[0].tobytes())
    bl[n >> 3] |= 1 << (n & 7)
    return (228 + len(cb)).to_bytes(4, "little") + serialize_attestation_data(att.data) + bytes(att.signature) + cb + bytes(bl)


def serialize_single_attestation(att: SingleAttestation) -> bytes:
    """SSZ wire form, 240 fixed bytes: [committee_index u64][attester_index u64][data][signature]."""
    return (int(att.committee_index).to_bytes(8, "little") + int(att.attester_index).to_bytes(8, "little") + serialize_attestation_data(att.data)
            + bytes(att.signature))


def serialize_aggregate_and_proof(m: AggregateAndProof) -> bytes:
    """SSZ: [aggregator_index u64][offset of aggregate = 108][selection_proof][Attestation]"""
    return int(m.aggregator_index).to_bytes(8, "little") + (108).to_bytes(4, "little") + bytes(m.selection_proof) + serialize_attestation(m.aggregate)


def serialize_signed_aggregate_and_proof(s: SignedAggregateAndProof) -> bytes:
    """SSZ: [offset of message = 100][signature][AggregateAndProof]"""
    return (100).to_bytes(4, "little") + bytes(s.signature) + serialize_aggregate_and_proof(s.message)


def serialize_sync_committee_message(m: SyncCommitteeMessage) -> bytes:
    """SSZ (:548-557): [slot u64][beacon_block_root][validator_index u64][signature], 144 bytes"""
    return int(m.slot).to_bytes(8, "little") + bytes(m.beacon_block_root) + int(m.validator_index).to_bytes(8, "little") + bytes(m.signature)


def serialize_signed_contribution_and_proof(s: SignedContributionAndProof) -> bytes:
    """SSZ, every field fixed (344 + ceil(len(aggregation_bits) / 8) bytes): [aggregator_index u64][slot u64][beacon_block_root]
    [subcommittee_index u64][aggregation_bits Bitvector][contribution signature][selection_proof][signature]"""
    m, c = s.message, s.message.contribution
    return (int(m.aggregator_index).to_bytes(8, "little") + int(c.slot).to_bytes(8, "little") + bytes(c.beacon_block_root)
            + int(c.subcommittee_index).to_bytes(8, "little") + pack_bits([list(c.aggregation_bits)])[0].tobytes() + bytes(c.signature)
            + bytes(m.selection_proof) + bytes(s.signature))


def serialize_validators(validators) -> np.ndarray:
    """SSZ serialisation of each Validator (:36-45) -> uint8[n, 121]: pubkey 48, withdrawal_credentials 32, effective_balance u64,
    slashed 1, activation_eligibility_epoch, activation_epoch, exit_epoch, withdrawable_epoch u64, little-endian.  The record format of
    Engine.ssz_validators_load / ssz_validators_update."""
    n = len(validators)
    out = np.zeros((n, 121), dtype=np.uint8)
    if n == 0:
        return out
    u64 = lambda f: np.array([getattr(v, f) for v in validators], dtype="<u8").view(np.uint8).reshape(n, 8)      # noqa: E731
    out[:, 0:48] = np.frombuffer(b"".join(bytes(v.pubkey) for v in validators), dtype=np.uint8).reshape(n, 48)
    out[:, 48:80] = np.frombuffer(b"".join(bytes(v.withdrawal_credentials) for v in validators), dtype=np.uint8).reshape(n, 32)
    out[:, 80:88] = u64("effective_balance")
    out[:, 88] = [1 if v.slashed else 0 for v in validators]
    for k, f in enumerate(("activation_eligibility_epoch", "activation_epoch", "exit_epoch", "withdrawable_epoch")):
        out[:, 89 + 8 * k:97 + 8 * k] = u64(f)
    return out


def _chunk_depth(limit: int, size: int) -> int:
    """depth of the chunk tree of `limit` basic values (or roots) of `size` bytes"""
    return ((limit * size + 31) // 32 - 1).bit_length()


def _pubkey_root(pk: bytes) -> bytes:
    """hash_tree_root(BLSPubkey): the 48 bytes in two chunks, the second zero-padded"""
    assert len(pk) == 48
    return sha256(bytes(pk) + bytes(16))


def compute_domain(domain_type: bytes, fork_version: bytes, genesis_validators_root: bytes) -> bytes:
    fork_data_root = _merkle([bytes(fork_version) + bytes(28), bytes(genesis_validators_root)])
    return bytes(domain_type) + fork_data_root[:28]


def integer_squareroot(n: int) -> int:
    x, y = n, (n + 1) // 2
    while y < x:
        x, y = y, (y + n // y) // 2
    return x


def shuffle_permutation(n: int, seed: bytes, rounds: int) -> np.ndarray:
    """perm[i] = compute_shuffled_index(i, n, seed) (:513-534) for every i at once: one pivot hash and
    ceil(n/256) source hashes per round instead of two hashes per index per round."""
    idx = np.arange(n, dtype=np.int64)
    if n == 0:
        return idx.astype(np.uint32)
    nblk = (n + 255) // 256
    for rnd in range(rounds):
        r = bytes([rnd])
        pivot = int.from_bytes(sha256(seed + r)[:8], "little") % n
        src = b"".join(sha256(seed + r + blk.to_bytes(4, "little")) for blk in range(nblk))
        bits = np.unpackbits(np.frombuffer(src, dtype=np.uint8), bitorder="little")
        flip = (pivot + n - idx) % n
        pos = np.maximum(idx, flip)
        idx = np.where(bits[pos] == 1, flip, idx)
    return idx.astype(np.uint32)


def pack_bits(rows, stride=None) -> np.ndarray:
    """list of bool lists -> uint8[n, stride], bit j of row a at byte j>>3, bit j&7 (SSZ Bitlist order)."""
    n = max((len(r) for r in rows), default=0)
    stride = stride or max(1, (n + 7) // 8)
    out = np.zeros((len(rows), stride), dtype=np.uint8)
    for a, r in enumerate(rows):
        if len(r):
            packed = np.packbits(np.asarray(r, dtype=np.uint8), bitorder="little")
            out[a, :packed.shape[0]] = packed
    return out


class Spec:
    """pyspec functions bound to a preset and a GPU engine."""

    def __init__(self, preset: Preset = MAINNET, engine: Engine = None, incremental_tree: bool = False):
        """incremental_tree: keep the device block tree current across new blocks and finalization (Engine.tree_add / tree_prune /
        tree_set_viable, rooted at the finalized block) instead of re-uploading the store whenever its blocks or checkpoints change
        (see _sync_store).  Heads and weights are the same either way."""
        self.p = preset
        self.engine = engine if engine is not None else Engine(0)
        self.incremental_tree = incremental_tree
        self._registry_key = None          # (length, fingerprint of the pubkey bytes) of the registry on the device
        self._balances_key = None          # (state object, slot) whose effective balances / flags are on the device
        self._balances_state = None
        self._committee_cache = {}
        self._mirror = None                # device mirror of a Store (block tree + latest messages), see _sync_store
        self.registry_valid = None         # KeyValidate verdict per validator of the registry on the device (uint8[n])
        self._sync_key = None              # (length, hash of the pubkey bytes) of the sync committee on the device
        self.sync_committee_valid = None   # KeyValidate verdict per position of that committee (uint8[SYNC_COMMITTEE_SIZE])
        self._sync_positions = None        # (registry and committee key, first registry index per position): _position_validators
        self._ssz_records = None           # serialised validators of the device tree of hash_tree_root_state (uint8[n, 121])
        self._ssz_load_id = None           # engine.ssz_loads after this Spec's last load: another load replaced the tree when it differs
        self._slasher = None               # slasher_start: size and current epoch of the device history, accepted attestations by target epoch
        self.stats = {"registry_uploads": 0, "balance_refreshes": 0, "store_uploads": 0, "lmd_device_updates": 0, "sync_committee_uploads": 0,
                      "ssz_validator_loads": 0, "ssz_validator_updates": 0, "tree_adds": 0, "tree_prunes": 0, "viability_updates": 0}
        # full: fingerprint = hash of ALL pubkeys on every call (O(n) host work, catches any in-place replacement);
        # sampled: first / last / 62 strided pubkeys (O(1)); auto: full up to 65 536 validators, sampled above
        self.registry_check = "auto"

    # ------------------------------------------------------------------ epochs / registry
    def compute_epoch_at_slot(self, slot):
        return slot // self.p.SLOTS_PER_EPOCH

    def compute_start_slot_at_epoch(self, epoch):
        return epoch * self.p.SLOTS_PER_EPOCH

    def get_current_epoch(self, state):
        return self.compute_epoch_at_slot(state.slot)

    def get_previous_epoch(self, state):
        cur = self.get_current_epoch(state)
        return GENESIS_EPOCH if cur == GENESIS_EPOCH else cur - 1

    @staticmethod
    def is_active_validator(v, epoch):
        return v.activation_epoch <= epoch < v.exit_epoch

    def get_active_validator_indices(self, state, epoch):
        return [i for i, v in enumerate(state.validators) if v.activation_epoch <= epoch < v.exit_epoch]

    def get_total_active_balance(self, state):
        e = self.get_current_epoch(state)
        tot = sum(v.effective_balance for v in state.validators if v.activation_epoch <= e < v.exit_epoch)
        return max(self.p.EFFECTIVE_BALANCE_INCREMENT, tot)

    def get_total_balance(self, state, indices):                             # described at :811
        return max(self.p.EFFECTIVE_BALANCE_INCREMENT, sum(state.validators[i].effective_balance for i in indices))

    @staticmethod
    def has_flag(flags: int, flag_index: int) -> bool:                          # ParticipationFlags helper used at :747
        return (int(flags) >> flag_index) & 1 == 1

    @staticmethod
    def add_flag(flags: int, flag_index: int) -> int:                           # :748
        return int(flags) | (1 << flag_index)

    def get_unslashed_participating_indices(self, state, flag_index, epoch):   # described at :805-807 (host set form)
        cur = self.get_current_epoch(state)
        assert epoch in (self.get_previous_epoch(state), cur)
        table = state.current_epoch_participation if epoch == cur else state.previous_epoch_participation
        return set(i for i in self.get_active_validator_indices(state, epoch)
                   if self.has_flag(table[i], flag_index) and not state.validators[i].slashed)

    # ------------------------------------------------------------------ FFG accounting (:793-803, :817-852)
    def process_justification_and_finalization(self, state):
        """:793-803.  The three balance sums (total active, previous / current epoch TIMELY_TARGET balance of unslashed
        validators) are one pass over the device registry and participation tables (b2_ffg_balances); the 2/3 tests and the
        four finalization rules are scalar host logic."""
        cur = self.get_current_epoch(state)
        if cur <= GENESIS_EPOCH + 1:
            return
        self.sync_registry(state)
        eng = self.engine
        eng.participation_load(0, np.asarray(state.current_epoch_participation, dtype=np.uint8))
        eng.participation_load(1, np.asarray(state.previous_epoch_participation, dtype=np.uint8))
        total, cur_target, prev_target, _ = eng.ffg_balances(TIMELY_TARGET_FLAG_INDEX)
        inc = self.p.EFFECTIVE_BALANCE_INCREMENT                                # get_total_balance's floor
        self.weigh_justification_and_finalization(state, max(inc, total), max(inc, prev_target), max(inc, cur_target))

    def weigh_justification_and_finalization(self, state, total_active_balance, previous_epoch_target_balance,
                                             current_epoch_target_balance):    # :817-852
        prev_epoch, cur_epoch = self.get_previous_epoch(state), self.get_current_epoch(state)
        old_prev, old_cur = state.previous_justified_checkpoint, state.current_justified_checkpoint
        state.previous_justified_checkpoint = old_cur
        bits = [0] + [int(b) for b in state.justification_bits[:JUSTIFICATION_BITS_LENGTH - 1]]
        for pos, epoch, balance in ((1, prev_epoch, previous_epoch_target_balance), (0, cur_epoch, current_epoch_target_balance)):
            if 3 * balance >= 2 * total_active_balance:                        # :830, :834
                state.current_justified_checkpoint = Checkpoint(epoch=epoch, root=self.get_block_root(state, epoch))
                bits[pos] = 1
        state.justification_bits = bits
        # :842-852 -- (bits [lo, hi) all set, source checkpoint, its distance from the current epoch), in the reference's order
        for lo, hi, source, dist in ((1, 4, old_prev, 3), (1, 3, old_prev, 2), (0, 3, old_cur, 2), (0, 2, old_cur, 1)):
            if all(bits[lo:hi]) and source.epoch + dist == cur_epoch:
                state.finalized_checkpoint = source

    def get_randao_mix(self, state, epoch):
        return state.randao_mixes[epoch % self.p.EPOCHS_PER_HISTORICAL_VECTOR]

    def get_block_root_at_slot(self, state, slot):
        assert slot < state.slot <= slot + self.p.SLOTS_PER_HISTORICAL_ROOT
        return state.block_roots[slot % self.p.SLOTS_PER_HISTORICAL_ROOT]

    def get_block_root(self, state, epoch):
        return self.get_block_root_at_slot(state, self.compute_start_slot_at_epoch(epoch))

    # ------------------------------------------------------------------ committees
    def get_committee_count_per_slot(self, state, epoch):                      # :461-468
        n_active = len(self.get_active_validator_indices(state, epoch))
        return max(1, min(self.p.MAX_COMMITTEES_PER_SLOT, n_active // self.p.SLOTS_PER_EPOCH // self.p.TARGET_COMMITTEE_SIZE))

    def get_seed(self, state, epoch, domain_type):                             # :481-486
        mix = self.get_randao_mix(state, epoch + self.p.EPOCHS_PER_HISTORICAL_VECTOR - self.p.MIN_SEED_LOOKAHEAD - 1)
        return sha256(domain_type + int(epoch).to_bytes(8, "little") + mix)

    def compute_shuffled_index(self, index, index_count, seed):                # :513-534 (per-index form)
        assert index < index_count
        for rnd in range(self.p.SHUFFLE_ROUND_COUNT):
            r = bytes([rnd])
            pivot = int.from_bytes(sha256(seed + r)[0:8], "little") % index_count
            flip = (pivot + index_count - index) % index_count
            position = max(index, flip)
            source = sha256(seed + r + (position // 256).to_bytes(4, "little"))
            if (source[(position % 256) // 8] >> (position % 8)) & 1:
                index = flip
        return index

    def compute_committee(self, indices, seed, index, count):                  # :495-504
        n = len(indices)
        start, end = (n * index) // count, (n * (index + 1)) // count
        perm = self._permutation(n, seed)
        return [indices[int(perm[i])] for i in range(start, end)]

    def _permutation(self, n, seed):
        key = (n, seed, self.p.SHUFFLE_ROUND_COUNT)
        if key not in self._committee_cache:
            if len(self._committee_cache) > 8:
                self._committee_cache.clear()
            if hasattr(self.engine, "shuffle_committees"):      # SHA-256 + swap-or-not rounds on the GPU (k_shuffle_*)
                self._committee_cache[key] = self.engine.shuffle_committees(seed, n, self.p.SHUFFLE_ROUND_COUNT)
            else:                                               # engine stand-ins of the CPU tests
                self._committee_cache[key] = shuffle_permutation(n, seed, self.p.SHUFFLE_ROUND_COUNT)
        return self._committee_cache[key]

    def epoch_committees(self, state, epoch):
        """All committees of ``epoch`` in array form: (members u32[n_active], off u32[count+1], committees_per_slot)."""
        active = np.asarray(self.get_active_validator_indices(state, epoch), dtype=np.uint32)
        cps = self.get_committee_count_per_slot(state, epoch)
        seed = self.get_seed(state, epoch, DOMAIN_BEACON_ATTESTER)
        n = len(active)
        members = active[self._permutation(n, seed)]
        count = cps * self.p.SLOTS_PER_EPOCH
        off = np.array([(n * k) // count for k in range(count + 1)], dtype=np.uint32)
        return members, off, cps

    def get_beacon_committee(self, state, slot, index):                        # called at :729
        epoch = self.compute_epoch_at_slot(slot)
        members, off, cps = self.epoch_committees(state, epoch)
        k = (slot % self.p.SLOTS_PER_EPOCH) * cps + index
        return members[off[k]:off[k + 1]].tolist()

    def compute_proposer_index(self, state, indices, seed):                    # :604-618
        assert len(indices) > 0
        i, total = 0, len(indices)
        while True:
            cand = indices[self.compute_shuffled_index(i % total, total, seed)]
            random_byte = sha256(seed + (i // 32).to_bytes(8, "little"))[i % 32]
            if state.validators[cand].effective_balance * 255 >= self.p.MAX_EFFECTIVE_BALANCE * random_byte:
                return cand
            i += 1

    def get_beacon_proposer_index(self, state):                                # called at :754
        epoch = self.get_current_epoch(state)
        seed = sha256(self.get_seed(state, epoch, DOMAIN_BEACON_PROPOSER) + int(state.slot).to_bytes(8, "little"))
        return self.compute_proposer_index(state, self.get_active_validator_indices(state, epoch), seed)

    # ------------------------------------------------------------------ signing
    def get_domain(self, state, domain_type, epoch=None):
        epoch = self.get_current_epoch(state) if epoch is None else epoch
        fv = state.fork.previous_version if epoch < state.fork.epoch else state.fork.current_version
        return compute_domain(domain_type, fv, state.genesis_validators_root)

    @staticmethod
    def compute_signing_root(data: AttestationData, domain):
        return _merkle([hash_tree_root_attestation_data(data), bytes(domain)])

    # ------------------------------------------------------------------ SSZ wire decode on the device (:714-717)
    def decode_attestations(self, encodings):
        """List of SSZ-encoded Attestations -> list of Attestation (None where the encoding is malformed: no delimiter bit, more
        than MAX_VALIDATORS_PER_COMMITTEE bits, truncated container).  One GPU call for the batch (b2_attestations_decode); the
        same call yields the bit rows and the 128-byte data records the verification kernels take."""
        if not encodings:
            return []
        limit = self.p.MAX_VALIDATORS_PER_COMMITTEE
        off = np.zeros(len(encodings) + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(e) for e in encodings])
        bits, blen, data, sig, st = self.engine.attestations_decode(b"".join(bytes(e) for e in encodings), off, (limit + 7) // 8, limit)
        out = []
        for a in range(len(encodings)):
            if st[a] != 0:
                out.append(None)
                continue
            row = np.unpackbits(bits[a], bitorder="little")[:int(blen[a])]
            out.append(Attestation([bool(x) for x in row], deserialize_attestation_data(data[a].tobytes()), sig[a].tobytes()))
        return out

    # ------------------------------------------------------------------ registry on the device
    def _pubkey_fingerprint(self, validators):
        n = len(validators)
        mode = self.registry_check
        if mode == "auto":
            mode = "full" if n <= 65536 else "sampled"
        h = hashlib.blake2b(digest_size=16)
        if mode == "full":
            h.update(b"".join(bytes(v.pubkey) for v in validators))
        else:
            step = max(1, n // 62)
            for i in list(range(0, n, step)) + [n - 1]:
                h.update(i.to_bytes(8, "little") + bytes(validators[i].pubkey))
        return h.digest()

    def invalidate_registry(self):
        """Forget what is on the device: the next call re-uploads the registry and the store (call it after replacing pubkeys in
        place in a registry larger than 65 536 validators, where the content check is sampled -- see registry_check)."""
        self._registry_key = self._balances_key = self._balances_state = self._mirror = None

    def sync_pubkeys(self, state):
        """state.validators[*].pubkey on the device.  Decompressed + KeyValidated on the GPU ONCE per registry CONTENT: the cache key is
        (length, fingerprint of the pubkey bytes), never an address -- so neither a recycled id() nor an in-place replacement can
        alias a stale registry, and two states that share the same validator set (the justified state and a target checkpoint
        state) share one upload.  Signature verification needs nothing else.  Returns True when it uploaded."""
        validators = state.validators
        n = len(validators)
        key = (n, self._pubkey_fingerprint(validators))
        if key == self._registry_key:
            return False
        pk = np.frombuffer(b"".join(bytes(v.pubkey) for v in validators), dtype=np.uint8).reshape(n, 48)
        zero = np.zeros(n, dtype=np.uint64)
        self.registry_valid = self.engine.registry_load(pk, zero, np.zeros(n, dtype=np.uint8))    # resets the device LMD table too
        self._registry_key = key
        self._balances_key = self._balances_state = self._mirror = None
        self.stats["registry_uploads"] += 1
        return True

    def sync_registry(self, state):
        """sync_pubkeys + the per-validator effective balance / activity / slashed table of THIS state (what the fork-choice weights
        and the FFG sums read).  Refreshed once per (state object, slot): the spec changes these fields only at epoch processing
        (:122-133) and in slashings; a different state (or slot) re-reads them (an O(n) pass over the Python objects)."""
        self.sync_pubkeys(state)
        bkey = (id(state), state.slot)
        if bkey == self._balances_key and state is self._balances_state:
            return
        validators = state.validators
        n = len(validators)
        epoch = self.get_current_epoch(state)
        eff = np.fromiter((v.effective_balance for v in validators), dtype=np.uint64, count=n)
        prev = self.get_previous_epoch(state)
        # bit0 active in the current epoch, bit1 slashed, bit2 active in the previous epoch (the FFG sums need both epochs)
        flags = np.fromiter(((1 if v.activation_epoch <= epoch < v.exit_epoch else 0) | (2 if v.slashed else 0)
                             | (4 if v.activation_epoch <= prev < v.exit_epoch else 0)
                             for v in validators), dtype=np.uint8, count=n)
        self.engine.registry_update_balances(eff, flags)
        self.stats["balance_refreshes"] += 1
        self._balances_key, self._balances_state = bkey, state                  # the state is held: its id() cannot be recycled
        self._total_active = (int(eff[(flags & 1) != 0].astype(object).sum()) if n else 0, int(np.count_nonzero(flags & 1)))

    # ------------------------------------------------------------------ indexed attestations (called at :736, :745, :975-976)
    def get_attesting_indices(self, state, data, bits):
        committee = self.get_beacon_committee(state, data.slot, data.index)
        return set(v for i, v in enumerate(committee) if bits[i])

    def get_indexed_attestation(self, state, attestation):
        idx = self.get_attesting_indices(state, attestation.data, attestation.aggregation_bits)
        return IndexedAttestation(sorted(idx), attestation.data, attestation.signature)

    def is_valid_indexed_attestation(self, state, indexed):
        return bool(self.are_valid_indexed_attestations(state, [indexed])[0])

    def are_valid_indexed_attestations(self, state, indexed_list):
        """Batched is_valid_indexed_attestation: one GPU FastAggregateVerify call for the whole list."""
        if not indexed_list:
            return np.zeros(0, dtype=np.uint8)
        self.sync_pubkeys(state)
        n = len(state.validators)
        members, off, sigs, structurally_ok, data128, domains = [], [0], [], [], [], []
        for ia in indexed_list:
            idx = list(ia.attesting_indices)
            good = len(idx) > 0 and idx == sorted(set(idx)) and idx[-1] < n and len(bytes(ia.signature)) == 96
            structurally_ok.append(good)
            members += idx if good else []
            off.append(len(members))
            domains.append(self.get_domain(state, DOMAIN_BEACON_ATTESTER, ia.data.target.epoch))
            data128.append(serialize_attestation_data(ia.data))
            sigs.append(bytes(ia.signature) if len(bytes(ia.signature)) == 96 else bytes(96))
        if hasattr(self.engine, "signing_roots"):           # SSZ merkleization on the GPU (k_signing_roots)
            msgs_arr = self.engine.signing_roots(np.frombuffer(b"".join(data128), dtype=np.uint8), np.frombuffer(b"".join(domains), dtype=np.uint8))
        else:
            msgs_arr = np.frombuffer(b"".join(self.compute_signing_root(ia.data, dom) for ia, dom in zip(indexed_list, domains)), dtype=np.uint8)
        sizes = np.diff(np.asarray(off, dtype=np.int64))
        stride = max(1, (int(sizes.max()) + 7) // 8)
        bits = np.zeros((len(indexed_list), stride), dtype=np.uint8)
        for a, s in enumerate(sizes):
            full, rem = divmod(int(s), 8)
            bits[a, :full] = 0xFF
            if rem:
                bits[a, full] = (1 << rem) - 1
        ok = self.engine.fast_aggregate_verify(np.asarray(members, dtype=np.uint32), off, bits,
                                               msgs_arr, np.frombuffer(b"".join(sigs), dtype=np.uint8))
        return ok & np.asarray(structurally_ok, dtype=np.uint8)

    # ------------------------------------------------------------------ participation helpers (called at :733, :747-754)
    def get_attestation_participation_flag_indices(self, state, data, inclusion_delay):
        justified = state.current_justified_checkpoint if data.target.epoch == self.get_current_epoch(state) else state.previous_justified_checkpoint
        matching_source = data.source == justified
        matching_target = matching_source and data.target.root == self.get_block_root(state, data.target.epoch)
        matching_head = matching_target and data.beacon_block_root == self.get_block_root_at_slot(state, data.slot)
        assert matching_source
        flags = []
        if matching_source and inclusion_delay <= integer_squareroot(self.p.SLOTS_PER_EPOCH):
            flags.append(TIMELY_SOURCE_FLAG_INDEX)
        if matching_target and inclusion_delay <= self.p.SLOTS_PER_EPOCH:
            flags.append(TIMELY_TARGET_FLAG_INDEX)
        if matching_head and inclusion_delay == self.p.MIN_ATTESTATION_INCLUSION_DELAY:
            flags.append(TIMELY_HEAD_FLAG_INDEX)
        return flags

    def get_base_reward_per_increment(self, state):
        return self.p.EFFECTIVE_BALANCE_INCREMENT * BASE_REWARD_FACTOR // integer_squareroot(self.get_total_active_balance(state))

    def get_base_reward(self, state, index):
        return (state.validators[index].effective_balance // self.p.EFFECTIVE_BALANCE_INCREMENT) * self.get_base_reward_per_increment(state)

    # ------------------------------------------------------------------ process_attestation (:722-754)
    def _check_attestation(self, state, attestation):
        data = attestation.data
        assert data.target.epoch in (self.get_previous_epoch(state), self.get_current_epoch(state))     # :724
        assert data.target.epoch == self.compute_epoch_at_slot(data.slot)                                # :725
        assert data.slot + self.p.MIN_ATTESTATION_INCLUSION_DELAY <= state.slot <= data.slot + self.p.SLOTS_PER_EPOCH   # :726
        assert data.index < self.get_committee_count_per_slot(state, data.target.epoch)                 # :727
        committee = self.get_beacon_committee(state, data.slot, data.index)                              # :729
        assert len(attestation.aggregation_bits) == len(committee)                                       # :730
        flag_indices = self.get_attestation_participation_flag_indices(state, data, state.slot - data.slot)
        return committee, flag_indices

    def _apply_attestation(self, state, attestation, committee, flag_indices):
        data = attestation.data
        participation = state.current_epoch_participation if data.target.epoch == self.get_current_epoch(state) else state.previous_epoch_participation
        per_inc = self.get_base_reward_per_increment(state)
        numerator = 0
        for v, bit in zip(committee, attestation.aggregation_bits):                                      # :745-749
            if not bit:
                continue
            for flag_index, weight in enumerate(PARTICIPATION_FLAG_WEIGHTS):
                if flag_index in flag_indices and not (participation[v] >> flag_index) & 1:
                    participation[v] |= 1 << flag_index
                    numerator += (state.validators[v].effective_balance // self.p.EFFECTIVE_BALANCE_INCREMENT) * per_inc * weight
        denominator = (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT) * WEIGHT_DENOMINATOR // PROPOSER_WEIGHT     # :752
        state.balances[self.get_beacon_proposer_index(state)] += numerator // denominator                # :753-754

    def process_attestation(self, state, attestation):
        committee, flag_indices = self._check_attestation(state, attestation)
        assert self.is_valid_indexed_attestation(state, self.get_indexed_attestation(state, attestation))   # :736 -> GPU
        self._apply_attestation(state, attestation, committee, flag_indices)

    def process_attestations(self, state, attestations):
        """process_operations' attestation loop with ONE GPU verification batch.  Same observable behaviour as calling
        process_attestation in order: the first invalid attestation raises AssertionError after its predecessors were applied."""
        pre = []
        for att in attestations:
            try:
                pre.append(self._check_attestation(state, att) + (self.get_indexed_attestation(state, att),))
            except AssertionError:
                pre.append(None)
                break
        verdicts = self.are_valid_indexed_attestations(state, [p[2] for p in pre if p is not None])
        n_ok = 0
        while n_ok < len(attestations) and n_ok < len(pre) and pre[n_ok] is not None and verdicts[n_ok]:
            n_ok += 1
        if n_ok and hasattr(self.engine, "participation_update"):
            self._apply_attestations_gpu(state, attestations[:n_ok], pre[:n_ok])
        else:
            for k in range(n_ok):
                self._apply_attestation(state, attestations[k], pre[k][0], pre[k][1])
        assert n_ok == len(attestations)

    def _apply_attestations_gpu(self, state, attestations, pre):
        """Flag scatter + proposer-reward numerators of :745-752 for a prefix of valid attestations on the GPU (order-exact),
        then the per-attestation integer division and the proposer credit of :752-754 on the host."""
        eng = self.engine
        self.sync_registry(state)              # the reward numerators read THIS state's effective balances on the device
        cur = self.get_current_epoch(state)
        tables = (state.current_epoch_participation, state.previous_epoch_participation)
        per_inc = self.get_base_reward_per_increment(state)
        denominator = (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT) * WEIGHT_DENOMINATOR // PROPOSER_WEIGHT
        proposer = self.get_beacon_proposer_index(state)
        for which in (0, 1):
            sel = [k for k, att in enumerate(attestations) if (att.data.target.epoch == cur) == (which == 0)]
            if not sel:
                continue
            members, off, rows, masks = [], [0], [], []
            for k in sel:
                members += pre[k][0]
                off.append(len(members))
                rows.append(attestations[k].aggregation_bits)
                masks.append(sum(1 << f for f in pre[k][1]))
            eng.participation_load(which, np.asarray(tables[which], dtype=np.uint8))
            num = eng.participation_update(which, np.asarray(members, dtype=np.uint32), off, pack_bits(rows), np.asarray(masks, dtype=np.uint8), None,
                                           self.p.EFFECTIVE_BALANCE_INCREMENT, per_inc)
            tables[which][:] = eng.participation_read(which).tolist()
            for v in num:
                state.balances[proposer] += int(v) // denominator

    def process_block_attestations(self, state, blocks):
        """process_attestation (:722-754) for every attestation of a run of consecutive blocks of the state's chain in one epoch, one GPU
        call (b2_block_attestations): state.slot == blocks[0].slot, the state as process_block sees the first block.  Block-atomic as
        on_block's state_transition (:1008-1009): the blocks before the first invalid one are applied in order (participation flags, and
        each block's proposer reward credited to its proposer_index), nothing of that block or of a later one.  The chain's roots below
        blocks[0].slot come from state.block_roots; block k's root stands for the slots [slot_k, slot_{k+1}).  state.slot and block_roots
        are left as they are.  Returns (n_applied, statuses): per block, the status (0-11, include/b200pos.h) of each attestation."""
        return self._process_block_attestations(state, blocks, self.block_attestations_inputs, self.engine.block_attestations)

    def _process_block_attestations(self, state, blocks, inputs, call):
        """both block-attestation calls: the arguments by inputs(state, blocks), the Engine method `call`, then the results into the state"""
        assert blocks and state.slot == blocks[0].slot
        block_off = np.concatenate([[0], np.cumsum([len(b.attestations) for b in blocks])]).astype(np.uint32)
        if not block_off[-1]:
            return len(blocks), [np.zeros(0, np.int32) for _ in blocks]
        args = inputs(state, blocks)
        self.sync_registry(state)              # first: a registry reload drops the device participation tables
        eng = self.engine
        eng.participation_load(0, np.asarray(state.current_epoch_participation, dtype=np.uint8))
        eng.participation_load(1, np.asarray(state.previous_epoch_participation, dtype=np.uint8))
        res = call(**args)
        if res.n_applied:
            state.current_epoch_participation[:] = eng.participation_read(0).tolist()
            state.previous_epoch_participation[:] = eng.participation_read(1).tolist()
            for k in range(res.n_applied):
                state.balances[blocks[k].proposer_index] += int(res.block_reward[k])
        return res.n_applied, [res.status[block_off[k]:block_off[k + 1]] for k in range(len(blocks))]

    def block_attestations_inputs(self, state, blocks):
        """The arguments of Engine.block_attestations for these blocks on this state (as process_block_attestations passes them): the
        attestations' encodings and offsets, the committees of epochs e - 1 and e, the chain's roots (state.block_roots below
        blocks[0].slot, block k's root for [slot_k, slot_{k+1})), the justified checkpoints, the attester domains and the scalars."""
        args = self._block_attestations_args(state, blocks, serialize_attestation)
        args["bits_stride"] = max(1, (int(np.diff(args["off"].astype(np.int64)).max()) + 7) // 8)
        return args

    def _block_attestations_args(self, state, blocks, serialize):
        """what both block-attestation calls take: the encodings by `serialize` and their offsets, the block rows and slots, the
        committees of epochs e - 1 and e, the chain's roots, the justified checkpoints, the attester domains and the scalars"""
        p = self.p
        spe = p.SLOTS_PER_EPOCH
        e = blocks[0].slot // spe
        mem_c, off_c, cps_c = self.epoch_committees(state, e)
        if e > 0:
            mem_p, off_p, cps_p = self.epoch_committees(state, e - 1)
            members = np.concatenate([mem_p, mem_c]).astype(np.uint32)
            off = np.concatenate([off_p[:-1], off_c + np.uint32(len(mem_p))]).astype(np.uint32)
        else:
            members, off, cps_p = mem_c, off_c, 0
        start = e * spe
        roots = []
        for s in range(start - spe, start + spe):
            if s < blocks[0].slot:
                roots.append(bytes(state.block_roots[s % p.SLOTS_PER_HISTORICAL_ROOT]) if s >= 0 else bytes(32))
            else:
                roots.append(bytes([b for b in blocks if b.slot <= s][-1].root))
        cps = lambda c: int(c.epoch).to_bytes(8, "little") + bytes(c.root)      # noqa: E731
        wires = [serialize(a) for b in blocks for a in b.attestations]
        return dict(wire=b"".join(wires), woff=np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32),
                    block_off=np.concatenate([[0], np.cumsum([len(b.attestations) for b in blocks])]).astype(np.uint32),
                    block_slot=np.array([b.slot for b in blocks], dtype=np.uint64), members=members, off=off, cps_prev=cps_p, cps_cur=cps_c,
                    chain_roots=np.frombuffer(b"".join(roots), dtype=np.uint8),
                    justified80=cps(state.previous_justified_checkpoint) + cps(state.current_justified_checkpoint),
                    domains64=self.get_domain(state, DOMAIN_BEACON_ATTESTER, max(e, 1) - 1) + self.get_domain(state, DOMAIN_BEACON_ATTESTER, e),
                    slots_per_epoch=spe, min_inclusion_delay=p.MIN_ATTESTATION_INCLUSION_DELAY, increment=p.EFFECTIVE_BALANCE_INCREMENT,
                    base_reward_per_increment=self.get_base_reward_per_increment(state))

    def process_block_attestations_electra(self, state, blocks):
        """process_block_attestations for blocks whose attestations are ElectraAttestations (one GPU call, b2_block_attestations_electra):
        Electra's process_attestation with Deneb's inclusion window and flags.  Block-atomic, the chain's roots, the proposers' rewards and
        what is left unchanged as in process_block_attestations.  Returns (n_applied, statuses): per block, the status (0-13,
        include/b200pos.h) of each attestation."""
        return self._process_block_attestations(state, blocks, self.block_attestations_electra_inputs, self.engine.block_attestations_electra)

    def block_attestations_electra_inputs(self, state, blocks):
        """The arguments of Engine.block_attestations_electra for these blocks of ElectraAttestations on this state: those of
        block_attestations_inputs with the Electra encodings, MAX_COMMITTEES_PER_SLOT and MAX_VALIDATORS_PER_COMMITTEE in place of bits_stride."""
        args = self._block_attestations_args(state, blocks, serialize_attestation_electra)
        args.update(max_committees_per_slot=self.p.MAX_COMMITTEES_PER_SLOT, max_validators_per_committee=self.p.MAX_VALIDATORS_PER_COMMITTEE)
        return args

    # ------------------------------------------------------------------ block packing (BeaconBlockBody.attestations :639, :659)
    def get_attestations_for_block(self, state, pool, max_attestations=None) -> List[Attestation]:
        """The attestations a proposer at state.slot includes: the pool entries process_attestation would accept (signatures are
        assumed gossip-validated and not verified here), disjoint aggregates of one AttestationData folded into one, then up to
        max_attestations (MAX_ATTESTATIONS) folded aggregates chosen greedily by proposer-reward numerator against the state's
        participation -- one GPU call (b2_pack_attestations).  Returned in pick order, ready for process_attestations."""
        max_out = self.p.MAX_ATTESTATIONS if max_attestations is None else int(max_attestations)
        committees, data_ids, datas = {}, {}, []
        members, off, table = [], [0], []
        cand_comm, cand_data, masks, rows, sigs = [], [], [], [], []
        cur = self.get_current_epoch(state)
        for att in pool:
            try:
                committee, flag_indices = self._check_attestation(state, att)
            except AssertionError:
                continue
            d = att.data
            k = committees.get((d.slot, d.index))
            if k is None:
                k = committees[(d.slot, d.index)] = len(table)
                members += committee
                off.append(len(members))
                table.append(0 if d.target.epoch == cur else 1)
            root = hash_tree_root_attestation_data(d)
            if root not in data_ids:
                data_ids[root] = len(datas)
                datas.append(d)
            cand_comm.append(k)
            cand_data.append(data_ids[root])
            masks.append(sum(1 << f for f in flag_indices))
            rows.append(att.aggregation_bits)
            sig = bytes(att.signature)
            sigs.append(sig if len(sig) == 96 else bytes(96))          # a wrong length never decodes
        if not rows or max_out <= 0:
            return []
        self.sync_registry(state)              # first: a registry reload drops the device participation tables
        eng = self.engine
        eng.participation_load(0, np.asarray(state.current_epoch_participation, dtype=np.uint8))
        eng.participation_load(1, np.asarray(state.previous_epoch_participation, dtype=np.uint8))
        sizes = np.diff(np.asarray(off, dtype=np.int64))
        res = eng.pack_attestations(np.asarray(members, dtype=np.uint32), off, table, cand_comm, cand_data, masks,
                                    pack_bits(rows, stride=max(1, (int(sizes.max()) + 7) // 8)), np.frombuffer(b"".join(sigs), dtype=np.uint8),
                                    max_out, self.p.EFFECTIVE_BALANCE_INCREMENT, self.get_base_reward_per_increment(state))
        out = []
        for o in range(len(res.committee)):
            n = int(sizes[int(res.committee[o])])
            row = np.unpackbits(res.bits[o], bitorder="little")[:n]
            out.append(Attestation([bool(x) for x in row], datas[int(res.data[o])], res.signature[o].tobytes()))
        return out

    # ------------------------------------------------------------------ sync committee (:371-372, :540-590; Altair)
    def compute_sync_committee_period(self, epoch):                            # :586-587
        return epoch // self.p.EPOCHS_PER_SYNC_COMMITTEE_PERIOD

    def is_assigned_to_sync_committee(self, state, epoch, validator_index):    # :564-577
        sync_committee_period = self.compute_sync_committee_period(epoch)
        current_sync_committee_period = self.compute_sync_committee_period(self.get_current_epoch(state))
        next_sync_committee_period = current_sync_committee_period + 1
        assert sync_committee_period in (current_sync_committee_period, next_sync_committee_period)
        pubkey = state.validators[validator_index].pubkey
        if sync_committee_period == current_sync_committee_period:
            return pubkey in state.current_sync_committee.pubkeys
        return pubkey in state.next_sync_committee.pubkeys

    def sync_committee_on_device(self, state):
        """state.current_sync_committee.pubkeys on the device, decoded, KeyValidated and summed ONCE per committee CONTENT (the cache key
        is the length and a hash of all the pubkey bytes, as sync_pubkeys keys the registry).  Returns True when it uploaded."""
        pubkeys = [bytes(pk) for pk in state.current_sync_committee.pubkeys]
        key = (len(pubkeys), hashlib.blake2b(b"".join(pubkeys), digest_size=16).digest())
        if key == self._sync_key:
            return False
        self._sync_key = None                  # a failed load below leaves nothing cached
        self.sync_committee_valid = self.engine.sync_committee_load(np.frombuffer(b"".join(pubkeys), dtype=np.uint8), len(pubkeys))
        self._sync_key = key
        self.stats["sync_committee_uploads"] += 1
        return True

    def verify_sync_aggregates(self, state, items):
        """eth_fast_aggregate_verify of state.current_sync_committee for a batch of (slot, block_root, SyncAggregate): signing root
        sha256(block_root || get_domain(state, DOMAIN_SYNC_COMMITTEE, compute_epoch_at_slot(slot))) -- one b2_sha256_batch call --
        and every verdict in one b2_sync_aggregate_verify call.  A bit vector of the wrong length or a signature that is not 96 bytes
        is False.  -> uint8[len(items)]"""
        if not items:
            return np.zeros(0, dtype=np.uint8)
        self.sync_committee_on_device(state)
        size = len(state.current_sync_committee.pubkeys)
        roots, rows, sigs, shape_ok = [], [], [], []
        for slot, block_root, agg in items:
            bits, sig = list(agg.sync_committee_bits), bytes(agg.sync_committee_signature)
            good = len(bits) == size and len(sig) == 96 and len(bytes(block_root)) == 32
            shape_ok.append(good)
            roots.append((bytes(block_root) if good else ZERO32) + self.get_domain(state, DOMAIN_SYNC_COMMITTEE, self.compute_epoch_at_slot(slot)))
            rows.append(bits if good else [])
            sigs.append(sig if good else bytes(96))
        msgs = self.engine.sha256_batch(np.frombuffer(b"".join(roots), dtype=np.uint8), 64)
        ok = self.engine.sync_aggregate_verify(np.zeros(len(items), dtype=np.uint32), pack_bits(rows, (size + 7) // 8), msgs,
                                               np.frombuffer(b"".join(sigs), dtype=np.uint8))
        return ok & np.asarray(shape_ok, dtype=np.uint8)

    def process_sync_aggregate(self, state, sync_aggregate):
        """Altair process_sync_aggregate, restated from the upstream consensus specs (specs/altair/beacon-chain.md; the reference
        names the sync committee but does not contain this function).  The signature check runs on the GPU against the cached
        committee (verify_sync_aggregates); the committee_size balance updates stay on the host."""
        previous_slot = max(state.slot, 1) - 1
        root = self.get_block_root_at_slot(state, previous_slot)
        assert self.verify_sync_aggregates(state, [(previous_slot, root, sync_aggregate)])[0]
        total_active_increments = self.get_total_active_balance(state) // self.p.EFFECTIVE_BALANCE_INCREMENT
        total_base_rewards = self.get_base_reward_per_increment(state) * total_active_increments
        max_participant_rewards = total_base_rewards * SYNC_REWARD_WEIGHT // WEIGHT_DENOMINATOR // self.p.SLOTS_PER_EPOCH
        participant_reward = max_participant_rewards // self.p.SYNC_COMMITTEE_SIZE
        proposer_reward = participant_reward * PROPOSER_WEIGHT // (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT)
        first = {}
        for i, v in enumerate(state.validators):                # all_pubkeys.index(pubkey): the FIRST registry index of a key
            first.setdefault(bytes(v.pubkey), i)
        committee_indices = []
        for pk in state.current_sync_committee.pubkeys:
            if bytes(pk) not in first:
                raise ValueError("sync committee pubkey is not in the registry")
            committee_indices.append(first[bytes(pk)])
        proposer = self.get_beacon_proposer_index(state)
        for participant_index, participation_bit in zip(committee_indices, sync_aggregate.sync_committee_bits):
            if participation_bit:
                state.balances[participant_index] += participant_reward
                state.balances[proposer] += proposer_reward
            else:
                state.balances[participant_index] = max(0, state.balances[participant_index] - participant_reward)

    def sync_committee_for_messages(self, state):
        """The committee compute_subnets_for_sync_committee (upstream Altair validator spec) reads: state.current_sync_committee, or
        state.next_sync_committee when state.slot + 1 starts the next sync committee period."""
        next_slot_epoch = self.compute_epoch_at_slot(state.slot + 1)
        if self.compute_sync_committee_period(self.get_current_epoch(state)) == self.compute_sync_committee_period(next_slot_epoch):
            return state.current_sync_committee
        return state.next_sync_committee

    def _position_validators(self, state, committee):
        """uint32[len(committee.pubkeys)]: the first registry index of each committee key (all_pubkeys.index(pubkey), as
        process_sync_aggregate maps positions), cached per (registry, committee) content"""
        pubkeys = [bytes(pk) for pk in committee.pubkeys]
        key = (self._registry_key, len(pubkeys), hashlib.blake2b(b"".join(pubkeys), digest_size=16).digest())
        if self._sync_positions is not None and self._sync_positions[0] == key:
            return self._sync_positions[1]
        first = {}
        for i, v in enumerate(state.validators):
            first.setdefault(bytes(v.pubkey), i)
        if any(pk not in first for pk in pubkeys):
            raise ValueError("sync committee pubkey is not in the registry")
        pv = np.array([first[pk] for pk in pubkeys], dtype=np.uint32)
        self._sync_positions = (key, pv)
        return pv

    def validate_sync_committee_messages(self, state, items, current_slot=None):
        """The sync_committee_{subnet_id} gossip checks (upstream Altair p2p spec) of one slot's list of (subnet_id, SyncCommitteeMessage) on
        the GPU (b2_sync_committee_messages), and the contributions and SyncAggregates process_sync_committee_contributions (upstream Altair
        validator spec) builds from the accepted ones.  current_slot defaults to state.slot; the committee is sync_committee_for_messages';
        the domain is get_domain(DOMAIN_SYNC_COMMITTEE) of current_slot's epoch, the epoch of every message that can be accepted.  Subnet
        membership compares registry indices, each committee key standing for its first registry index.  Returns (status per item, 0-6 of
        include/b200pos.h; the present SyncCommitteeContributions in (root, subnet) order, roots by first accepted message; a SyncAggregates
        {root: SyncAggregate}).  Each call starts with an empty seen-cache."""
        current_slot = state.slot if current_slot is None else int(current_slot)
        self.sync_registry(state)
        committee = self.sync_committee_for_messages(state)
        size, count = len(committee.pubkeys), self.p.SYNC_COMMITTEE_SUBNET_COUNT
        aggregates = SyncAggregates(size)
        if not items:
            return [], [], aggregates
        pv = self._position_validators(state, committee)
        wires = [serialize_sync_committee_message(m) for _, m in items]
        woff = np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)
        subnet = np.array([int(sid) if 0 <= int(sid) < 2**32 else 2**32 - 1 for sid, _ in items], dtype=np.uint32)
        domain = self.get_domain(state, DOMAIN_SYNC_COMMITTEE, self.compute_epoch_at_slot(current_slot))
        r = self.engine.sync_committee_messages(b"".join(wires), woff, subnet, pv, count, current_slot, domain)
        sub = size // count
        contributions = []
        for k in range(r.roots.shape[0]):
            root = r.roots[k].tobytes()
            for sc in range(count):
                if r.contrib_present[k, sc]:
                    bits = np.unpackbits(r.contrib_bits[k, sc], bitorder="little")[:sub]
                    contributions.append(SyncCommitteeContribution(current_slot, root, sc, [bool(b) for b in bits], r.contrib_sigs[k, sc].tobytes()))
            aggregates[root] = SyncAggregate([bool(b) for b in np.unpackbits(r.agg_bits[k], bitorder="little")[:size]], r.agg_sigs[k].tobytes())
        return [int(x) for x in r.status], contributions, aggregates

    def validate_sync_contribution_and_proofs(self, state, items, current_slot=None):
        """The sync_committee_contribution_and_proof gossip checks (upstream Altair p2p spec) of one slot's list of SignedContributionAndProof
        on the GPU (b2_sync_contribution_and_proof_intake), and per root the SyncAggregate process_sync_committee_contributions (upstream
        Altair validator spec) builds from its best accepted contribution per subnet.  current_slot defaults to state.slot; the committee is
        sync_committee_for_messages' (get_sync_subcommittee_pubkeys' rule: the next committee when state.slot + 1 starts a new period); the
        domains are those of current_slot's epoch.  Subcommittee membership compares registry indices, each committee key standing for its
        first registry index.  Returns (status per item, 0-12 of include/b200pos.h; a SyncAggregates {root: SyncAggregate}, the empty
        aggregate for a root with no accepted contribution).  Each call starts with empty seen-caches."""
        current_slot = state.slot if current_slot is None else int(current_slot)
        self.sync_registry(state)
        committee = self.sync_committee_for_messages(state)
        size, count = len(committee.pubkeys), self.p.SYNC_COMMITTEE_SUBNET_COUNT
        aggregates = SyncAggregates(size)
        if not items:
            return [], aggregates
        pv = self._position_validators(state, committee)
        wires = [serialize_signed_contribution_and_proof(x) for x in items]
        woff = np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)
        epoch = self.compute_epoch_at_slot(current_slot)
        domains = b"".join(self.get_domain(state, d, epoch) for d in (DOMAIN_SYNC_COMMITTEE, DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF,
                                                                      DOMAIN_CONTRIBUTION_AND_PROOF))
        r = self.engine.sync_contribution_and_proof_intake(b"".join(wires), woff, pv, count, current_slot, domains,
                                                           self.p.TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE)
        for k in range(r.roots.shape[0]):
            bits = np.unpackbits(r.agg_bits[k], bitorder="little")[:size]
            aggregates[r.roots[k].tobytes()] = SyncAggregate([bool(b) for b in bits], r.agg_sigs[k].tobytes())
        return [int(x) for x in r.status], aggregates

    # ------------------------------------------------------------------ fork choice
    def update_latest_messages(self, store, attesting_indices, attestation):   # :1435-1441
        """The store's dict is updated as the reference does; when the store is mirrored on the device (after a get_head /
        get_weight call) the same update is applied to the device table by K7 (b2_latest_messages_update), so the next get_head
        is a kernel launch, not a re-upload."""
        target, root = attestation.data.target, attestation.data.beacon_block_root
        indices = [int(i) for i in attesting_indices]
        for i in indices:
            if i in store.equivocating_indices:
                continue
            if i not in store.latest_messages or target.epoch > store.latest_messages[i].epoch:
                store.latest_messages[i] = LatestMessage(epoch=target.epoch, root=root)
        m = self._mirror
        if m is not None and m["store"] is store:
            if self.incremental_tree and root not in m["index"] and root in store.blocks:
                self._sync_blocks(store, m)          # a vote for a block on_block added since the last get_head
            blk = m["index"].get(root) if self._mirror is m else None
            if blk is None or not indices or max(indices) >= m["n_val"] or target.epoch >= 0xFFFFFFFF:
                self._mirror = None                  # a vote the device form cannot hold: fall back to a full re-upload
            else:
                k = len(indices)
                bits = np.full((1, (k + 7) // 8), 0xFF, dtype=np.uint8)
                if k & 7:
                    bits[0, -1] = (1 << (k & 7)) - 1
                self.engine.latest_messages_update(np.asarray(indices, dtype=np.uint32), [0, k], bits, [target.epoch], [blk])
                m["n_msgs"] = len(store.latest_messages)
                self.stats["lmd_device_updates"] += 1

    def get_current_slot(self, store):
        return (store.time - store.genesis_time) // getattr(self.p, "SECONDS_PER_SLOT", 12)

    def get_ancestor(self, store, root, slot):
        block = store.blocks[root]
        while block.slot > slot:
            root = block.parent_root
            block = store.blocks[root]
        return root

    def validate_on_attestation(self, store, attestation, is_from_block):      # called at :970 (upstream fork-choice spec, v1.2.0)
        target = attestation.data.target
        if not is_from_block:                                                   # validate_target_epoch_against_current_time
            current_epoch = self.compute_epoch_at_slot(self.get_current_slot(store))
            previous_epoch = current_epoch - 1 if current_epoch > GENESIS_EPOCH else GENESIS_EPOCH
            assert target.epoch in (current_epoch, previous_epoch)
        assert target.epoch == self.compute_epoch_at_slot(attestation.data.slot)
        assert target.root in store.blocks
        assert attestation.data.beacon_block_root in store.blocks
        assert store.blocks[attestation.data.beacon_block_root].slot <= attestation.data.slot
        assert target.root == self.get_ancestor(store, attestation.data.beacon_block_root, self.compute_start_slot_at_epoch(target.epoch))
        assert self.get_current_slot(store) >= attestation.data.slot + 1

    def on_attestation(self, store, attestation, is_from_block=False):         # :963-979 / :1423-1428
        """AssertionError = invalid, as in the reference.  store_target_checkpoint_state (:971) needs process_slots, which is state
        transition and out of scope (DESIGN.md section 7): the target checkpoint state must already be in store.checkpoint_states
        (the caller's on_block / on_tick put it there), otherwise the attestation is rejected."""
        self.validate_on_attestation(store, attestation, is_from_block)
        assert attestation.data.target in store.checkpoint_states, "target checkpoint state not in store (store_target_checkpoint_state is out of scope)"
        target_state = store.checkpoint_states[attestation.data.target]
        indexed = self.get_indexed_attestation(target_state, attestation)
        assert self.is_valid_indexed_attestation(target_state, indexed)
        self.update_latest_messages(store, indexed.attesting_indices, attestation)

    def validate_aggregate_and_proofs(self, state, store, items, current_slot=None):
        """The beacon_aggregate_and_proof gossip checks (upstream phase 0 p2p spec) of a list of SignedAggregateAndProof on the GPU
        (b2_aggregate_and_proof_intake).  Returns (status per item, the accepted items' Attestations in list order): statuses 0-20 of
        include/b200pos.h, where an item whose data.slot lies neither in current_slot's epoch nor in the one before it gets 7.  The items
        are split by the epoch of data.slot, one call per epoch, committees from `state`; each call starts with empty seen-caches.
        Needs Spec(incremental_tree=True): its device tree is rooted at the finalized block, so "not in the tree" also covers the
        IGNORE for a finalized checkpoint that is not an ancestor."""
        if not self.incremental_tree:
            raise ValueError("validate_aggregate_and_proofs needs Spec(incremental_tree=True): the device tree must be rooted at the finalized block")
        current_slot = self.get_current_slot(store) if current_slot is None else int(current_slot)
        self._sync_store(store)
        self.sync_registry(state)
        status = [7] * len(items)
        cur = self.compute_epoch_at_slot(current_slot)
        for epoch in [cur] + ([cur - 1] if cur > GENESIS_EPOCH else []):
            sel = [i for i, x in enumerate(items) if self.compute_epoch_at_slot(x.message.aggregate.data.slot) == epoch]
            if not sel:
                continue
            wires = [serialize_signed_aggregate_and_proof(items[i]) for i in sel]
            woff = np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)
            members, off, cps = self.epoch_committees(state, epoch)
            stride = max(1, (int(np.diff(off.astype(np.int64)).max()) + 7) // 8)      # the bit rows of the epoch's largest committee
            domains = b"".join(self.get_domain(state, d, epoch) for d in (DOMAIN_BEACON_ATTESTER, DOMAIN_SELECTION_PROOF, DOMAIN_AGGREGATE_AND_PROOF))
            r = self.engine.aggregate_and_proof_intake(b"".join(wires), woff, members, off, epoch, current_slot, domains, cps, self.p.SLOTS_PER_EPOCH,
                                                       stride, self.p.TARGET_AGGREGATORS_PER_COMMITTEE, self.p.ATTESTATION_PROPAGATION_SLOT_RANGE)
            for k, i in enumerate(sel):
                status[i] = int(r.status[k])
        return status, [items[i].message.aggregate for i in range(len(items)) if status[i] == 0]

    @staticmethod
    def is_slashable_attestation_data(data_1, data_2):                         # :1134-1143
        double_vote = data_1 != data_2 and data_1.target.epoch == data_2.target.epoch
        surround_vote = data_1.source.epoch < data_2.source.epoch and data_2.target.epoch < data_1.target.epoch
        return double_vote or surround_vote

    def on_attester_slashing(self, store, attester_slashing):                  # :1447-1461
        a1, a2 = attester_slashing.attestation_1, attester_slashing.attestation_2
        assert self.is_slashable_attestation_data(a1.data, a2.data)
        state = store.block_states[store.justified_checkpoint.root]
        ok = self.are_valid_indexed_attestations(state, [a1, a2])              # both signatures in one GPU batch
        assert ok[0] and ok[1]
        both = sorted(set(a1.attesting_indices).intersection(a2.attesting_indices))
        for index in both:
            store.equivocating_indices.add(index)
        m = self._mirror
        if m is not None and m["store"] is store:
            if hasattr(self.engine, "on_attester_slashing") and both and both[-1] < m["n_val"]:
                self.engine.on_attester_slashing(both, both)                    # mark them on the device table as well
                m["n_equiv"] = len(store.equivocating_indices)
            else:
                self._mirror = None

    # ------------------------------------------------------------------ slashing detection (:1128-1143 -> AttesterSlashing :1160-1162)
    def slasher_start(self, state, history_epochs, max_attestations_per_target=None):
        """Start a slasher (Engine.slasher_init) for the validators of `state` at its current epoch: a device-resident history of
        history_epochs epochs that find_attester_slashings feeds.  max_attestations_per_target defaults to twice the committees of an epoch."""
        per_target = max_attestations_per_target or 2 * self.p.MAX_COMMITTEES_PER_SLOT * self.p.SLOTS_PER_EPOCH
        cur = self.get_current_epoch(state)
        self.engine.slasher_init(len(state.validators), history_epochs, per_target, cur)
        self._slasher = dict(n=len(state.validators), H=int(history_epochs), cur=cur, recorded={})

    def find_attester_slashings(self, state, indexed_attestations, verify=True) -> List[AttesterSlashing]:
        """Offer IndexedAttestations to the slasher and return the AttesterSlashings they complete, against everything offered before and
        against each other.  verify: only attestations that pass is_valid_indexed_attestation(state, .) are recorded.  The double and
        surround votes are found on the GPU (b2_slasher_update); the host keeps the accepted attestations by target epoch inside the
        window and, only when something was flagged, looks up the partner at the reported target epoch, asserts
        is_slashable_attestation_data on the pair and orders it as on_attester_slashing wants it (attestation_1 surrounds attestation_2)."""
        sl = self._slasher
        assert sl is not None, "slasher_start first"
        atts = list(indexed_attestations)
        if not atts:
            return []
        n = sl["n"]
        accept = self.are_valid_indexed_attestations(state, atts) if verify else np.ones(len(atts), dtype=np.uint8)
        accept = np.array(accept, dtype=np.uint8)
        cur = self.get_current_epoch(state)
        if cur > sl["cur"]:
            self.engine.slasher_advance(cur)
            sl["cur"] = cur
            low = max(0, cur - sl["H"] + 1)
            for t in [t for t in sl["recorded"] if t < low]:      # nothing the device still accepts can conflict with them
                del sl["recorded"][t]
        members, off, src, tgt, roots = [], [0], [], [], []
        for a, ia in enumerate(atts):
            idx = [int(i) for i in ia.attesting_indices]
            s, t = int(ia.data.source.epoch), int(ia.data.target.epoch)
            if not (idx and idx == sorted(set(idx)) and idx[-1] < n and max(s, t) < 0xFFFFFFFF):
                accept[a], idx, s, t = 0, [], 0, 0              # what the device tables cannot hold is not offered
            members += idx
            off.append(len(members))
            src.append(s)
            tgt.append(t)
            roots.append(hash_tree_root_attestation_data(ia.data))
        sizes = np.diff(np.asarray(off, dtype=np.int64))
        bits = np.zeros((len(atts), max(1, (int(sizes.max()) + 7) // 8)), dtype=np.uint8)
        for a, k in enumerate(sizes):
            bits[a] = np.packbits(np.arange(8 * bits.shape[1]) < k, bitorder="little")
        status, kind, conflict, n_flagged = self.engine.slasher_update(
            np.asarray(members, dtype=np.uint32), off, bits, src, tgt, np.frombuffer(b"".join(roots), dtype=np.uint8), accept)
        for a in np.nonzero(status == 0)[0]:
            sl["recorded"].setdefault(tgt[a], []).append(atts[a])
        if n_flagged == 0:
            return []
        rules = {       # kind bit -> (partner's target epoch, ordered pair) of attestation `ia` with partner `c`
            1: lambda ia, c: ia.data != c.data and (c, ia),
            2: lambda ia, c: ia.data.source.epoch < c.data.source.epoch and (ia, c),
            4: lambda ia, c: c.data.source.epoch < ia.data.source.epoch and (c, ia),
        }
        out, seen = [], set()
        for i in np.nonzero(kind)[0]:
            a = int(np.searchsorted(off, i, side="right")) - 1
            ia, v = atts[a], members[i]
            for bit, target in ((1, tgt[a]), (2, int(conflict[i, 0])), (4, int(conflict[i, 1]))):
                if not kind[i] & bit:
                    continue
                pair = next(p for p in (rules[bit](ia, c) for c in sl["recorded"][target] if c is not ia and v in c.attesting_indices) if p)
                assert self.is_slashable_attestation_data(pair[0].data, pair[1].data)
                if (id(pair[0]), id(pair[1])) not in seen:
                    seen.add((id(pair[0]), id(pair[1])))
                    out.append(AttesterSlashing(pair[0], pair[1]))
        return out

    def _tree_root(self, store):
        """The root of the incremental device tree: the finalized checkpoint's block when the justified block descends from it, else
        the justified block (a store whose checkpoints are not on one chain)."""
        froot, jroot = store.finalized_checkpoint.root, store.justified_checkpoint.root
        r = jroot
        while froot in store.blocks and r in store.blocks and store.blocks[r].slot > store.blocks[froot].slot:
            r = store.blocks[r].parent_root
        return froot if r == froot else jroot

    def _store_arrays(self, store, root=None):
        """Store (dicts) -> the array form of include/b200pos.h: `root` (default: the justified root) and the blocks below it in
        topological order."""
        import collections
        root = store.justified_checkpoint.root if root is None else root
        children = {}
        for r, b in store.blocks.items():
            children.setdefault(b.parent_root, []).append(r)
        order, queue = [], collections.deque([root])
        while queue:
            r = queue.popleft()
            order.append(r)
            queue.extend(children.get(r, []))
        index = {r: i for i, r in enumerate(order)}
        nb = len(order)
        parent = np.zeros(nb, dtype=np.uint32)
        slot = np.zeros(nb, dtype=np.uint64)
        viable = np.ones(nb, dtype=np.uint8)
        for i, r in enumerate(order):
            b = store.blocks[r]
            slot[i] = b.slot
            if i:
                parent[i] = index[b.parent_root]
            if r not in children:
                viable[i] = self._leaf_viable(store, r)
        roots = np.frombuffer(b"".join(order), dtype=np.uint8).reshape(nb, 32)
        return order, index, parent, slot, roots, viable

    @staticmethod
    def _leaf_viable(store, root):                                             # the leaf test of get_filtered_block_tree (:1104)
        hs = store.block_states[root]
        cj = store.justified_checkpoint.epoch == GENESIS_EPOCH or hs.current_justified_checkpoint == store.justified_checkpoint
        cf = store.finalized_checkpoint.epoch == GENESIS_EPOCH or hs.finalized_checkpoint == store.finalized_checkpoint
        return 1 if (cj and cf) else 0

    def _sync_blocks(self, store, m):
        """incremental_tree: bring the device tree up to store.blocks without a reload.  The blocks on_block added since the last call
        (in store order, so parents first) are appended with one tree_add; a finalized checkpoint that moved to a block of the tree is
        applied with tree_prune, whose map re-numbers the mirror (the device re-maps the latest messages itself).  Blocks that do not
        descend from the tree's root are not mirrored.  A finalized block outside the tree drops the mirror (full reload)."""
        index, order, kids = m["index"], m["order"], m["kids"]
        if len(store.blocks) != m["n_seen"]:
            par, slot, roots, via = [], [], [], []
            for r, b in list(store.blocks.items())[m["n_seen"]:]:
                if r in index or b.parent_root not in index:
                    continue
                p = index[b.parent_root]
                index[r] = len(order)
                order.append(r)
                kids.append(0)
                kids[p] += 1
                par.append(p)
                slot.append(b.slot)
                roots.append(r)
                via.append(self._leaf_viable(store, r))
            m["n_seen"] = len(store.blocks)
            if par:
                self.engine.tree_add(par, slot, np.frombuffer(b"".join(roots), dtype=np.uint8), via)
                m["viable"].update(zip(range(len(order) - len(par), len(order)), via))
                m["boost"] = None
                self.stats["tree_adds"] += 1
        if store.finalized_checkpoint != m["finalized"]:
            froot = store.finalized_checkpoint.root
            if froot not in index:
                self._mirror = None
                return
            if index[froot] != 0:
                mp = self.engine.tree_prune(index[froot])
                keep = np.nonzero(mp != 0xFFFFFFFF)[0]
                m["order"] = order = [order[i] for i in keep]
                m["index"] = {r: i for i, r in enumerate(order)}
                m["kids"] = [kids[i] for i in keep]
                m["viable"] = {int(mp[i]): v for i, v in m["viable"].items() if mp[i] != 0xFFFFFFFF}
                m["boost"] = None
                self.stats["tree_prunes"] += 1
            m["finalized"] = store.finalized_checkpoint

    def _refresh_viability(self, store, m):
        """incremental_tree: every leaf's test reads the checkpoints, so when they move the leaves whose byte changed are sent"""
        cps = (store.justified_checkpoint, store.finalized_checkpoint)
        if m["checkpoints"] == cps:
            return
        m["checkpoints"] = cps
        changed = []
        for i, r in enumerate(m["order"]):
            if m["kids"][i] == 0:
                v = self._leaf_viable(store, r)
                if m["viable"].get(i) != v:
                    m["viable"][i] = v
                    changed.append((i, v))
        if changed:
            idx, val = zip(*changed)
            self.engine.tree_set_viable(idx, val)
            self.stats["viability_updates"] += 1

    def _sync_store(self, store):
        """Device mirror of the store: block tree (b2_tree_load) and latest messages (b2_latest_messages_load) are uploaded for another
        store object, a registry change, or latest_messages / equivocating_indices changed behind this class's back (their sizes differ
        from what the mirror recorded).  Without incremental_tree they are also uploaded when the justified / finalized checkpoint moved
        or a block was added (on_block); the tree is then rooted at the justified block.  With incremental_tree the tree is rooted at
        the finalized block: new blocks, finalization and leaf viability are applied on the device (_sync_blocks, _refresh_viability)
        and the latest messages are never re-uploaded for them; a justified block outside the tree, or a vote for a block the tree
        does not hold, falls back to the full upload.  Votes that arrive through on_attestation / update_latest_messages are applied
        to the device table incrementally, so between blocks get_head / get_weight cost one kernel sequence.
        Returns (order, index, justified block id, boost id, boost score)."""
        state = store.checkpoint_states[store.justified_checkpoint]
        self.sync_registry(state)
        m = self._mirror
        inc = self.incremental_tree
        live = (m is not None and m["store"] is store and m["n_msgs"] == len(store.latest_messages) and m["n_equiv"] == len(store.equivocating_indices)
                and m["n_val"] == len(state.validators))
        if live and not inc:
            live = m["justified"] == store.justified_checkpoint and m["finalized"] == store.finalized_checkpoint and m["n_seen"] == len(store.blocks)
        if live and inc:
            self._sync_blocks(store, m)
            live = self._mirror is m and store.justified_checkpoint.root in m["index"]
        if not live:
            order, index, parent, slot, roots, via = self._store_arrays(store, self._tree_root(store) if inc else None)
            self.engine.tree_load(parent, slot, roots, via)
            n = len(state.validators)
            epoch = np.zeros(n, dtype=np.uint64)
            blk = np.zeros(n, dtype=np.uint32)
            has = np.zeros(n, dtype=np.uint8)
            for v, lm in store.latest_messages.items():
                if v < n and lm.root in index:
                    epoch[v], blk[v], has[v] = lm.epoch, index[lm.root], 1
            eq = np.zeros(n, dtype=np.uint8)
            for v in store.equivocating_indices:
                if v < n:
                    eq[v] = 1
            self.engine.latest_messages_load(epoch, blk, has, eq)
            kids = np.bincount(parent[1:], minlength=len(order)).tolist()
            m = self._mirror = dict(store=store, justified=store.justified_checkpoint, finalized=store.finalized_checkpoint, n_seen=len(store.blocks),
                                    n_msgs=len(store.latest_messages), n_equiv=len(store.equivocating_indices), n_val=n, order=order, index=index,
                                    kids=kids, viable={i: int(via[i]) for i in range(len(order)) if kids[i] == 0},
                                    checkpoints=(store.justified_checkpoint, store.finalized_checkpoint), boost=None)
            self.stats["store_uploads"] += 1
        if inc:
            self._refresh_viability(store, m)
        bkey = (store.proposer_boost_root, self._balances_key)
        if m["boost"] is None or m["boost"][0] != bkey:
            boost_idx, boost_score = -1, 0
            if store.proposer_boost_root != ZERO32 and store.proposer_boost_root in m["index"]:
                total, num = self._total_active                                 # of the justified state, computed by sync_registry
                avg = max(self.p.EFFECTIVE_BALANCE_INCREMENT, total) // num
                boost_score = (num // self.p.SLOTS_PER_EPOCH) * avg * self.p.PROPOSER_SCORE_BOOST // 100
                boost_idx = m["index"][store.proposer_boost_root]
            m["boost"] = (bkey, boost_idx, boost_score)
        return m["order"], m["index"], m["index"][store.justified_checkpoint.root], m["boost"][1], m["boost"][2]

    def get_latest_attesting_balance(self, store, root):                       # called at :1116 (v1.2.0 form)
        order, index, justified, boost_idx, boost_score = self._sync_store(store)
        return int(self.engine.get_weights(boost_idx, boost_score)[index[root]])

    get_weight = get_latest_attesting_balance

    def get_head(self, store):                                                 # :1102-1116
        order, index, justified, boost_idx, boost_score = self._sync_store(store)
        return order[self.engine.get_head(justified, boost_idx, boost_score)]

    # ------------------------------------------------------------------ hash_tree_root(state) (:423, :1078)
    def validators_root(self, state) -> bytes:
        """hash_tree_root(state.validators) from the device tree: the records are diffed against those of the previous call and only
        the changed ones are sent as an update; a registry of another size, or a tree another caller loaded since, is re-loaded."""
        rec = serialize_validators(state.validators)
        old = self._ssz_records
        if old is None or old.shape[0] != rec.shape[0] or self.engine.ssz_loads != self._ssz_load_id:
            root = self.engine.ssz_validators_load(rec)
            self._ssz_load_id = self.engine.ssz_loads
            self.stats["ssz_validator_loads"] += 1
        else:
            idx = np.flatnonzero((old != rec).any(axis=1)).astype(np.uint32)
            root = self.engine.ssz_validators_update(idx, rec[idx])
            self.stats["ssz_validator_updates"] += 1
        self._ssz_records = rec
        return root

    def hash_tree_root_state(self, state) -> bytes:
        """hash_tree_root of the Bellatrix BeaconState (:338-374): its 25 field roots, padded to 32 leaves.  The validators, the other
        registry-sized lists and the large vectors are merkleized on the GPU; the small fields on the host.  A vector field left as
        None and a sync committee left as None hash as their SSZ default (all zero)."""
        p, eng = self.p, self.engine
        limit = p.VALIDATOR_REGISTRY_LIMIT

        def roots(values, length, depth, as_list=False):       # Vector / List of 32-byte roots
            values = [ZERO32] * length if values is None else values
            assert as_list or len(values) == length
            data = np.frombuffer(b"".join(bytes(r) for r in values), dtype=np.uint8)
            return eng.ssz_chunks_root(data, depth, len(values) if as_list else None)

        def basic_list(values, dtype):
            a = np.asarray(values, dtype=dtype)
            return eng.ssz_chunks_root(a, _chunk_depth(limit, a.itemsize), len(a))

        def sync_committee(c):
            pks, agg = ([bytes(48)] * p.SYNC_COMMITTEE_SIZE, bytes(48)) if c is None else (c.pubkeys, c.aggregate_pubkey)
            return _merkle([_merkle([_pubkey_root(pk) for pk in pks]), _pubkey_root(agg)])

        slashings = np.zeros(p.EPOCHS_PER_SLASHINGS_VECTOR, dtype="<u8") if state.slashings is None else np.asarray(state.slashings, dtype="<u8")
        assert slashings.shape == (p.EPOCHS_PER_SLASHINGS_VECTOR,)
        h, e1, x = state.latest_block_header, state.eth1_data, state.latest_execution_payload_header
        eth1_root = lambda e: _merkle([bytes(e.deposit_root), _u64_chunk(e.deposit_count), bytes(e.block_hash)])     # noqa: E731
        payload_header = _merkle([
            bytes(x.parent_hash), bytes(x.fee_recipient).ljust(32, b"\0"), bytes(x.state_root), bytes(x.receipts_root),
            _merkle([bytes(x.logs_bloom)[i:i + 32] for i in range(0, 256, 32)]), bytes(x.prev_randao), _u64_chunk(x.block_number),
            _u64_chunk(x.gas_limit), _u64_chunk(x.gas_used), _u64_chunk(x.timestamp),
            sha256(bytes(x.extra_data).ljust(32, b"\0") + len(x.extra_data).to_bytes(32, "little")),      # ByteList[32]: one chunk
            int(x.base_fee_per_gas).to_bytes(32, "little"), bytes(x.block_hash), bytes(x.transactions_root)])
        votes = np.frombuffer(b"".join(eth1_root(v) for v in state.eth1_data_votes), dtype=np.uint8)
        justification = sum(1 << i for i, b in enumerate(state.justification_bits) if b)
        fields = [
            _u64_chunk(state.genesis_time),
            bytes(state.genesis_validators_root),
            _u64_chunk(state.slot),
            _merkle([bytes(state.fork.previous_version).ljust(32, b"\0"), bytes(state.fork.current_version).ljust(32, b"\0"),
                     _u64_chunk(state.fork.epoch)]),
            _merkle([_u64_chunk(h.slot), _u64_chunk(h.proposer_index), bytes(h.parent_root), bytes(h.state_root), bytes(h.body_root)]),
            roots(state.block_roots, p.SLOTS_PER_HISTORICAL_ROOT, _chunk_depth(p.SLOTS_PER_HISTORICAL_ROOT, 32)),
            roots(state.state_roots, p.SLOTS_PER_HISTORICAL_ROOT, _chunk_depth(p.SLOTS_PER_HISTORICAL_ROOT, 32)),
            roots(state.historical_roots, None, _chunk_depth(p.HISTORICAL_ROOTS_LIMIT, 32), as_list=True),
            eth1_root(e1),
            eng.ssz_chunks_root(votes, _chunk_depth(p.EPOCHS_PER_ETH1_VOTING_PERIOD * p.SLOTS_PER_EPOCH, 32), len(state.eth1_data_votes)),
            _u64_chunk(state.eth1_deposit_index),
            self.validators_root(state),
            basic_list(state.balances, "<u8"),
            roots(state.randao_mixes, p.EPOCHS_PER_HISTORICAL_VECTOR, _chunk_depth(p.EPOCHS_PER_HISTORICAL_VECTOR, 32)),
            eng.ssz_chunks_root(slashings, _chunk_depth(p.EPOCHS_PER_SLASHINGS_VECTOR, 8)),
            basic_list(state.previous_epoch_participation, np.uint8),
            basic_list(state.current_epoch_participation, np.uint8),
            justification.to_bytes(32, "little"),
            hash_tree_root_checkpoint(state.previous_justified_checkpoint),
            hash_tree_root_checkpoint(state.current_justified_checkpoint),
            hash_tree_root_checkpoint(state.finalized_checkpoint),
            basic_list(state.inactivity_scores, "<u8"),
            sync_committee(state.current_sync_committee),
            sync_committee(state.next_sync_committee),
            payload_header,
        ]
        return _merkle(fields)
