"""hash_tree_root of the Bellatrix BeaconState and its parts -- CPU oracle (TEST INFRASTRUCTURE), hashlib only.

An independent restatement of the SSZ merkleization rules (SURVEY.md appendix C.3) for the fields of BeaconState (pos-evolution.md:338-374):
basic values are little-endian and packed into 32-byte chunks; a vector's root is the Merkle root of its chunks padded with zero chunks
to a power of two; a list's tree is padded to the chunk count of its limit and its root mixed with the length; a container's root is the
Merkle root of its field roots.  Containers the reference names without defining (BeaconBlockHeader, Eth1Data, ExecutionPayloadHeader,
SyncCommittee) follow upstream Bellatrix.  Objects are read by attribute, so the product's dataclasses can be passed in.
"""
import bisect
import hashlib

ZERO32 = bytes(32)
MAX_DEPTH = 64


def sha256(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()


def _zero_hashes():
    z = [ZERO32]
    for _ in range(MAX_DEPTH):
        z.append(sha256(z[-1] + z[-1]))
    return z


ZERO_HASHES = _zero_hashes()        # ZERO_HASHES[l] = root of 2^l zero chunks


def next_pow2(n: int) -> int:
    return 1 << max(n - 1, 0).bit_length()


def merkleize(chunks, limit=None) -> bytes:
    """Merkle root of the chunks padded with zero chunks to next_pow2(limit) (to next_pow2(len) without a limit).  The padding is
    virtual: a level with an odd node count is completed with the zero hash of that level."""
    n = len(chunks)
    width = next_pow2(n if limit is None else limit)
    assert n <= width
    depth = width.bit_length() - 1
    layer = list(chunks)
    for l in range(depth):
        if len(layer) % 2:
            layer.append(ZERO_HASHES[l])
        layer = [sha256(layer[i] + layer[i + 1]) for i in range(0, len(layer), 2)]
    return layer[0] if layer else ZERO_HASHES[depth]


def mix_in_length(root: bytes, length: int) -> bytes:
    return sha256(root + int(length).to_bytes(32, "little"))


def pack(data: bytes):
    """bytes -> 32-byte chunks, the last one zero-padded"""
    return [data[i:i + 32].ljust(32, b"\0") for i in range(0, len(data), 32)]


def uint_root(v: int, size: int = 8) -> bytes:
    return int(v).to_bytes(size, "little").ljust(32, b"\0")


def basic_vector_root(values, size: int) -> bytes:
    return merkleize(pack(b"".join(int(v).to_bytes(size, "little") for v in values)))


def basic_list_root(values, size: int, limit: int) -> bytes:
    data = b"".join(int(v).to_bytes(size, "little") for v in values)
    return mix_in_length(merkleize(pack(data), (limit * size + 31) // 32), len(values))


def roots_vector_root(roots) -> bytes:
    return merkleize([bytes(r) for r in roots])


def roots_list_root(roots, limit: int) -> bytes:
    return mix_in_length(merkleize([bytes(r) for r in roots], limit), len(roots))


def bitvector_root(bits) -> bytes:
    out = bytearray((len(bits) + 7) // 8)
    for i, b in enumerate(bits):
        if b:
            out[i >> 3] |= 1 << (i & 7)
    return merkleize(pack(bytes(out)) or [ZERO32])


def byte_list_root(data: bytes, limit: int) -> bytes:
    return mix_in_length(merkleize(pack(bytes(data)), (limit + 31) // 32), len(data))


def pubkey_root(pk: bytes) -> bytes:
    return merkleize(pack(bytes(pk)))


# ---- containers
def checkpoint_root(c) -> bytes:
    return merkleize([uint_root(c.epoch), bytes(c.root)])


def fork_root(f) -> bytes:
    return merkleize([bytes(f.previous_version).ljust(32, b"\0"), bytes(f.current_version).ljust(32, b"\0"), uint_root(f.epoch)])


def validator_root(v) -> bytes:
    return merkleize([pubkey_root(v.pubkey), bytes(v.withdrawal_credentials), uint_root(v.effective_balance), uint_root(int(bool(v.slashed)), 1),
                      uint_root(v.activation_eligibility_epoch), uint_root(v.activation_epoch), uint_root(v.exit_epoch),
                      uint_root(v.withdrawable_epoch)])


def serialize_validator(v) -> bytes:
    u = lambda x: int(x).to_bytes(8, "little")       # noqa: E731
    return (bytes(v.pubkey) + bytes(v.withdrawal_credentials) + u(v.effective_balance) + bytes([int(bool(v.slashed))])
            + u(v.activation_eligibility_epoch) + u(v.activation_epoch) + u(v.exit_epoch) + u(v.withdrawable_epoch))


def record_root(r: bytes) -> bytes:
    """hash_tree_root(Validator) of its 121-byte serialisation"""
    u = lambda o: uint_root(int.from_bytes(r[o:o + 8], "little"))      # noqa: E731
    return merkleize([pubkey_root(r[0:48]), r[48:80], u(80), uint_root(r[88], 1), u(89), u(97), u(105), u(113)])


def records_root(records, limit: int = 2**40) -> bytes:
    """hash_tree_root(List[Validator, limit]) of serialised records"""
    return mix_in_length(merkleize([record_root(r) for r in records], limit), len(records))


def block_header_root(h) -> bytes:
    return merkleize([uint_root(h.slot), uint_root(h.proposer_index), bytes(h.parent_root), bytes(h.state_root), bytes(h.body_root)])


def eth1_data_root(e) -> bytes:
    return merkleize([bytes(e.deposit_root), uint_root(e.deposit_count), bytes(e.block_hash)])


def execution_payload_header_root(h) -> bytes:
    return merkleize([bytes(h.parent_hash), bytes(h.fee_recipient).ljust(32, b"\0"), bytes(h.state_root), bytes(h.receipts_root),
                      merkleize(pack(bytes(h.logs_bloom))), bytes(h.prev_randao), uint_root(h.block_number), uint_root(h.gas_limit),
                      uint_root(h.gas_used), uint_root(h.timestamp), byte_list_root(h.extra_data, 32), uint_root(h.base_fee_per_gas, 32),
                      bytes(h.block_hash), bytes(h.transactions_root)])


def sync_committee_root(pubkeys, aggregate_pubkey) -> bytes:
    return merkleize([merkleize([pubkey_root(pk) for pk in pubkeys]), pubkey_root(aggregate_pubkey)])


def validators_root(validators, limit: int = 2**40) -> bytes:
    return mix_in_length(merkleize([validator_root(v) for v in validators], limit), len(validators))


def sparse_list_root(n: int, default_leaf: bytes, overrides: dict, limit: int) -> bytes:
    """Root of a list of n leaf roots, all default_leaf except overrides {index: root}, in O(len(overrides) * depth) hashes: a subtree
    inside the list without an override is the memoised default subtree of its height, one past the end a zero subtree."""
    keys = sorted(overrides)
    default = [default_leaf]
    depth = (next_pow2(limit)).bit_length() - 1
    for _ in range(depth):
        default.append(sha256(default[-1] + default[-1]))

    def node(level, i):
        lo, hi = i << level, (i + 1) << level
        if lo >= n:
            return ZERO_HASHES[level]
        j = bisect.bisect_left(keys, lo)
        if hi <= n and (j == len(keys) or keys[j] >= hi):
            return default[level]
        if level == 0:
            return overrides.get(i, default_leaf)
        return sha256(node(level - 1, 2 * i) + node(level - 1, 2 * i + 1))

    return mix_in_length(node(depth, 0), n)


# ---- BeaconState (Bellatrix, :338-374)
def state_root(state, preset) -> bytes:
    """preset: attributes SLOTS_PER_HISTORICAL_ROOT, EPOCHS_PER_HISTORICAL_VECTOR, EPOCHS_PER_SLASHINGS_VECTOR, SLOTS_PER_EPOCH,
    EPOCHS_PER_ETH1_VOTING_PERIOD, HISTORICAL_ROOTS_LIMIT, VALIDATOR_REGISTRY_LIMIT, SYNC_COMMITTEE_SIZE.  A vector field given as None
    and a sync committee given as None stand for their SSZ default value (all zero)."""
    p = preset
    limit = p.VALIDATOR_REGISTRY_LIMIT

    def vec(roots, length):
        roots = [ZERO32] * length if roots is None else roots
        assert len(roots) == length
        return roots_vector_root(roots)

    def sync(c):
        if c is None:
            return sync_committee_root([bytes(48)] * p.SYNC_COMMITTEE_SIZE, bytes(48))
        return sync_committee_root(c.pubkeys, c.aggregate_pubkey)

    slashings = [0] * p.EPOCHS_PER_SLASHINGS_VECTOR if state.slashings is None else state.slashings
    assert len(slashings) == p.EPOCHS_PER_SLASHINGS_VECTOR
    fields = [
        uint_root(state.genesis_time),
        bytes(state.genesis_validators_root),
        uint_root(state.slot),
        fork_root(state.fork),
        block_header_root(state.latest_block_header),
        vec(state.block_roots, p.SLOTS_PER_HISTORICAL_ROOT),
        vec(state.state_roots, p.SLOTS_PER_HISTORICAL_ROOT),
        roots_list_root(state.historical_roots, p.HISTORICAL_ROOTS_LIMIT),
        eth1_data_root(state.eth1_data),
        mix_in_length(merkleize([eth1_data_root(e) for e in state.eth1_data_votes], p.EPOCHS_PER_ETH1_VOTING_PERIOD * p.SLOTS_PER_EPOCH),
                      len(state.eth1_data_votes)),
        uint_root(state.eth1_deposit_index),
        validators_root(state.validators, limit),
        basic_list_root(state.balances, 8, limit),
        vec(state.randao_mixes, p.EPOCHS_PER_HISTORICAL_VECTOR),
        basic_vector_root(slashings, 8),
        basic_list_root(state.previous_epoch_participation, 1, limit),
        basic_list_root(state.current_epoch_participation, 1, limit),
        bitvector_root(state.justification_bits),
        checkpoint_root(state.previous_justified_checkpoint),
        checkpoint_root(state.current_justified_checkpoint),
        checkpoint_root(state.finalized_checkpoint),
        basic_list_root(state.inactivity_scores, 8, limit),
        sync(state.current_sync_committee),
        sync(state.next_sync_committee),
        execution_payload_header_root(state.latest_execution_payload_header),
    ]
    assert len(fields) == 25
    return merkleize(fields)
