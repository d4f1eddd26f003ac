"""Sync committees on the CPU oracle (TEST INFRASTRUCTURE): the Altair bls helpers eth_aggregate_pubkeys / eth_fast_aggregate_verify,
the SyncCommittee / SyncAggregate containers, the sync preset values, and compute_sync_committee_period, is_assigned_to_sync_committee
and process_sync_aggregate, built on oracle.bls_sig and oracle.spec (left as they are).

compute_sync_committee_period and is_assigned_to_sync_committee are the reference's (pos-evolution.md:564-587), restated here and
pinned to the reference's own text by tests/golden/literal_sync.json.  The reference names the sync committee (:371-372, :540-546) but
does not contain process_sync_aggregate or the two bls helpers: they are restated from the upstream consensus specs
(specs/altair/beacon-chain.md, specs/altair/bls.md), as recalled, not copied:
  * eth_aggregate_pubkeys: assert a non-empty list and KeyValidate of every key; the sum of the keys;
  * eth_fast_aggregate_verify: True for no keys and the G2 infinity signature, otherwise FastAggregateVerify;
  * process_sync_aggregate: previous_slot = max(state.slot, 1) - 1; signing root = hash_tree_root(SigningData(block root at previous_slot,
    get_domain(DOMAIN_SYNC_COMMITTEE, epoch of previous_slot))); assert eth_fast_aggregate_verify over the participants; then
    participant_reward = base_reward_per_increment * total active increments * SYNC_REWARD_WEIGHT // WEIGHT_DENOMINATOR // SLOTS_PER_EPOCH
    // SYNC_COMMITTEE_SIZE, proposer_reward = participant_reward * PROPOSER_WEIGHT // (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT); each
    participant (committee index = FIRST registry index of its key) gains participant_reward and the proposer proposer_reward, each
    non-participant loses participant_reward, floored at 0.
"""
import hashlib
from dataclasses import dataclass
from typing import List

from oracle import bls_sig as B
from oracle import spec as S
from oracle.bls12_381 import E1, g1_compress, g1_decompress

DOMAIN_SYNC_COMMITTEE = bytes.fromhex("07000000")
SYNC_REWARD_WEIGHT = 2
G2_POINT_AT_INFINITY = bytes([0xC0]) + bytes(95)
# preset name -> (SYNC_COMMITTEE_SIZE, EPOCHS_PER_SYNC_COMMITTEE_PERIOD)
SYNC_PRESET = {"mainnet": (512, 256), "minimal": (32, 8)}


@dataclass
class SyncCommittee:
    pubkeys: List[bytes]
    aggregate_pubkey: bytes


@dataclass
class SyncAggregate:
    sync_committee_bits: List[bool]
    sync_committee_signature: bytes


def eth_aggregate_pubkeys(pubkeys) -> bytes:
    assert len(pubkeys) > 0
    assert all(B.KeyValidate(pk) for pk in pubkeys)
    acc = E1.INF
    for pk in pubkeys:
        acc = E1.add(acc, g1_decompress(bytes(pk)))
    return g1_compress(acc)


def eth_fast_aggregate_verify(pubkeys, message: bytes, signature: bytes) -> bool:
    if len(pubkeys) == 0 and bytes(signature) == G2_POINT_AT_INFINITY:
        return True
    return B.FastAggregateVerify(pubkeys, message, signature)


class SyncSpec(S.Spec):
    """oracle.spec.Spec plus the sync-committee functions; states carry current_sync_committee / next_sync_committee attributes."""

    def __init__(self, preset=S.MAINNET, bls_module=B):
        super().__init__(preset, bls_module)
        self.SYNC_COMMITTEE_SIZE, self.EPOCHS_PER_SYNC_COMMITTEE_PERIOD = SYNC_PRESET[preset.name]

    def compute_sync_committee_period(self, epoch):                            # ref :586-587
        return epoch // self.EPOCHS_PER_SYNC_COMMITTEE_PERIOD

    def is_assigned_to_sync_committee(self, state, epoch, validator_index):    # ref :564-577
        period = self.compute_sync_committee_period(epoch)
        current = self.compute_sync_committee_period(self.get_current_epoch(state))
        assert period in (current, current + 1)
        pubkey = state.validators[validator_index].pubkey
        if period == current:
            return pubkey in state.current_sync_committee.pubkeys
        return pubkey in state.next_sync_committee.pubkeys

    def sync_signing_root(self, state, slot, block_root):
        """compute_signing_root(block_root, get_domain(state, DOMAIN_SYNC_COMMITTEE, compute_epoch_at_slot(slot))): the hash tree root
        of SigningData(object_root, domain) = sha256 of the two 32-byte chunks"""
        domain = self.get_domain(state, DOMAIN_SYNC_COMMITTEE, self.compute_epoch_at_slot(slot))
        return hashlib.sha256(bytes(block_root) + bytes(domain)).digest()

    def process_sync_aggregate(self, state, sync_aggregate):                   # upstream Altair
        committee_pubkeys = state.current_sync_committee.pubkeys
        participant_pubkeys = [pk for pk, bit in zip(committee_pubkeys, sync_aggregate.sync_committee_bits) if bit]
        previous_slot = max(state.slot, 1) - 1
        signing_root = self.sync_signing_root(state, previous_slot, self.get_block_root_at_slot(state, previous_slot))
        assert eth_fast_aggregate_verify(participant_pubkeys, signing_root, sync_aggregate.sync_committee_signature)
        total_active_increments = self.get_total_active_balance(state) // self.p.EFFECTIVE_BALANCE_INCREMENT
        total_base_rewards = self.get_base_reward_per_increment(state) * total_active_increments
        max_participant_rewards = total_base_rewards * SYNC_REWARD_WEIGHT // S.WEIGHT_DENOMINATOR // self.p.SLOTS_PER_EPOCH
        participant_reward = max_participant_rewards // self.SYNC_COMMITTEE_SIZE
        proposer_reward = participant_reward * S.PROPOSER_WEIGHT // (S.WEIGHT_DENOMINATOR - S.PROPOSER_WEIGHT)
        all_pubkeys = [v.pubkey for v in state.validators]
        committee_indices = [all_pubkeys.index(pubkey) for pubkey in committee_pubkeys]
        for participant_index, participation_bit in zip(committee_indices, sync_aggregate.sync_committee_bits):
            if participation_bit:
                self.increase_balance(state, participant_index, participant_reward)
                self.increase_balance(state, self.get_beacon_proposer_index(state), proposer_reward)
            else:
                state.balances[participant_index] = 0 if participant_reward > state.balances[participant_index] \
                    else state.balances[participant_index] - participant_reward


def minimal_sync_state(n_validators: int = 64, slot: int = 9, pks=None):
    """(SyncSpec, state) on the minimal preset with a current and a next sync committee: the current one repeats validator 3 at
    positions 1 and 2 (a duplicate member).  The third value is the validator index at each position of the current committee"""
    import scenarios
    pks = pks if pks is not None else scenarios.pubkeys(n_validators)
    spec, state = scenarios.minimal_state(n_validators, slot=slot, pks=pks)
    spec = SyncSpec(spec.p)
    size = spec.SYNC_COMMITTEE_SIZE
    cur = [(5 * i) % n_validators for i in range(size)]     # the same selections as tests/golden/gen_golden_sync.py
    cur[1] = cur[2] = 3
    nxt = [(7 * i + 11) % n_validators for i in range(size)]
    state.current_sync_committee = SyncCommittee([pks[i] for i in cur], eth_aggregate_pubkeys([pks[i] for i in cur]))
    state.next_sync_committee = SyncCommittee([pks[i] for i in nxt], eth_aggregate_pubkeys([pks[i] for i in nxt]))
    return spec, state, cur


def honest_sync_aggregate(spec, state, committee, bits):
    """SyncAggregate over the block root at max(state.slot, 1) - 1, signed by the secret keys of the participating positions
    (summed with multiplicity); the G2 infinity encoding when nobody participates"""
    import scenarios
    prev = max(state.slot, 1) - 1
    msg = spec.sync_signing_root(state, prev, spec.get_block_root_at_slot(state, prev))
    signers = [v for v, b in zip(committee, bits) if b]
    return SyncAggregate(list(bits), scenarios.sign_aggregate(signers, msg) if signers else G2_POINT_AT_INFINITY), msg
