"""Sync committees on the CPU oracle (tests/sync_oracle.py): compute_sync_committee_period and is_assigned_to_sync_committee against
what the reference's own text computes (tests/golden/literal_sync.json), the empty-participation rule of eth_fast_aggregate_verify,
eth_aggregate_pubkeys, and process_sync_aggregate's laws: an honest aggregate is accepted, a flipped bit is rejected, and the balances
move exactly as its reward formula says."""
import copy
import json
import os

import pytest

import bls_cases as bc
import scenarios
import sync_oracle as SO
from oracle import bls_sig as B
from oracle import spec as S
from oracle.bls12_381 import E1, g1_compress, g1_decompress

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "literal_sync.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def env():
    return SO.minimal_sync_state()


def test_literal_period_and_assignment(env, golden):
    spec, state, cur = env
    assert golden["preset"] == "minimal" and golden["current_sync_committee"] == cur
    assert len(cur) != len(set(cur))                                          # the golden committee holds a duplicate member
    for e, p in golden["period"].items():
        assert spec.compute_sync_committee_period(int(e)) == p
    st = copy.copy(state)
    n_assert = 0
    for case in golden["assigned"]:
        st.slot = case["state_slot"]
        if case["result"] == "assert":
            n_assert += 1
            with pytest.raises(AssertionError):
                spec.is_assigned_to_sync_committee(st, case["epoch"], 0)
        else:
            assert [spec.is_assigned_to_sync_committee(st, case["epoch"], v) for v in range(golden["n_validators"])] == case["result"], case
    assert n_assert and n_assert < len(golden["assigned"])


def test_eth_fast_aggregate_verify_empty_rule():
    M = bc.MSG
    pks = [B.SkToPk(bc.sk(k)) for k in (1, 2)]
    sig = bc.sign(bc.sk(1) + bc.sk(2))
    assert SO.eth_fast_aggregate_verify([], M, SO.G2_POINT_AT_INFINITY) is True
    assert SO.G2_POINT_AT_INFINITY == bc.INF2
    for other in (sig, bytes(96), bc.INF2[:95] + b"\x01", bytes([0xE0]) + bytes(95)):
        assert SO.eth_fast_aggregate_verify([], M, other) is False
    assert SO.eth_fast_aggregate_verify(pks, M, sig) is True
    neg = g1_compress(E1.neg(g1_decompress(pks[0])))
    assert SO.eth_fast_aggregate_verify([pks[0], neg], M, bc.INF2) is False      # keys that cancel are not "no keys"
    assert SO.eth_fast_aggregate_verify(pks, M, bc.INF2) is False


def test_eth_aggregate_pubkeys():
    pks = [B.SkToPk(bc.sk(k)) for k in (1, 2, 2)]
    assert SO.eth_aggregate_pubkeys(pks) == B.AggregatePKs(pks)
    for bad in ([], [pks[0], bc.INF1], [pks[0], bytes(48)]):
        with pytest.raises(AssertionError):
            SO.eth_aggregate_pubkeys(bad)


def _expected_balances(spec, state, cur, bits):
    total = spec.get_total_active_balance(state) // spec.p.EFFECTIVE_BALANCE_INCREMENT
    pr = spec.get_base_reward_per_increment(state) * total * SO.SYNC_REWARD_WEIGHT // S.WEIGHT_DENOMINATOR // spec.p.SLOTS_PER_EPOCH \
        // spec.SYNC_COMMITTEE_SIZE
    prop = pr * S.PROPOSER_WEIGHT // (S.WEIGHT_DENOMINATOR - S.PROPOSER_WEIGHT)
    out = list(state.balances)
    proposer = spec.get_beacon_proposer_index(state)
    for v, b in zip(cur, bits):
        if b:
            out[v] += pr
            out[proposer] += prop
        else:
            out[v] = max(0, out[v] - pr)
    return out, pr, prop


@pytest.mark.parametrize("pattern", ["all", "none", "first_half", "dup_only_one"])
def test_process_sync_aggregate_laws(env, pattern):
    spec, state, cur = env
    n = spec.SYNC_COMMITTEE_SIZE
    bits = {"all": [1] * n, "none": [0] * n, "first_half": [1] * (n // 2) + [0] * (n - n // 2),
            "dup_only_one": [1, 1, 0] + [1] * (n - 3)}[pattern]
    agg, _ = SO.honest_sync_aggregate(spec, state, cur, bits)
    st = copy.deepcopy(state)
    want, pr, prop = _expected_balances(spec, state, cur, bits)
    assert pr > 0 and prop > 0
    spec.process_sync_aggregate(st, agg)
    assert st.balances == want
    if pattern != "none":
        flipped = list(bits)
        flipped[5] ^= 1
        st = copy.deepcopy(state)
        with pytest.raises(AssertionError):
            spec.process_sync_aggregate(st, SO.SyncAggregate(flipped, agg.sync_committee_signature))
        assert st.balances == state.balances


def test_process_sync_aggregate_floor_and_first_index():
    """a non-participant whose balance is below the reward ends at 0; a key registered twice is credited at its FIRST index"""
    pks = scenarios.pubkeys(64)
    pks[40] = pks[3]                                                          # validator 40 re-uses validator 3's key
    spec, state, cur = SO.minimal_sync_state(pks=pks)
    state.balances[0] = 1
    bits = [0] + [1] * (spec.SYNC_COMMITTEE_SIZE - 1)
    first = [3 if v == 40 else v for v in cur]                                # the position of validator 40 holds key 3: secret key 3
    assert cur[0] == 0 and 40 in cur
    agg, _ = SO.honest_sync_aggregate(spec, state, first, bits)
    st = copy.deepcopy(state)
    spec.process_sync_aggregate(st, agg)
    want, _, _ = _expected_balances(spec, state, first, bits)
    assert st.balances == want and st.balances[0] == 0 and st.balances[40] == state.balances[40] != st.balances[3]
