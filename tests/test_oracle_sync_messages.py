"""Sync committee messages on the CPU: tests/sync_messages_oracle.py against the upstream rules it restates -- each contribution passes
eth_fast_aggregate_verify over its subnet's committee keys, each SyncAggregate passes process_sync_aggregate on the next slot's state, a
validator counts once per position it holds, the list-order seen rule -- and Spec.validate_sync_committee_messages' committee choice and
output form with a stub engine."""
import copy

import numpy as np
import pytest

import scenarios
import sync_messages_oracle as M
from oracle import bls_sig as B
from pos_evolution_b200 import spec as PS
from pos_evolution_b200.engine import SyncMessagesResult
from sync_oracle import SyncCommittee, eth_aggregate_pubkeys, eth_fast_aggregate_verify, minimal_sync_state

N_VAL, SLOT = 64, 9
ROOT_B = bytes(range(32))


@pytest.fixture(scope="module")
def setup():
    pks = scenarios.pubkeys(N_VAL)
    spec, state, cur = minimal_sync_state(N_VAL, slot=SLOT, pks=pks)
    cur = list(cur)
    cur[20] = cur[12]                       # one validator on subnets 1 and 2; validator 3 holds positions 1 and 2 (subnet 0)
    state.current_sync_committee = SyncCommittee([pks[v] for v in cur], eth_aggregate_pubkeys([pks[v] for v in cur]))
    domain = spec.get_domain(state, PS.DOMAIN_SYNC_COMMITTEE, spec.compute_epoch_at_slot(SLOT))
    return spec, state, cur, pks, domain


ROOT_A = scenarios._h(b"b200pos/blockroot" + SLOT.to_bytes(8, "little"))      # the state's block root at SLOT


def _scenario(cur, domain):
    """positions 24-31 on ROOT_B, the rest on ROOT_A"""
    wires, subnets, expect = M.scenario(cur, domain, SLOT, [ROOT_A, ROOT_B], lambda p: int(p >= 24), N_VAL)
    return wires, subnets, expect, ROOT_A


@pytest.fixture(scope="module")
def run(setup):
    spec, state, cur, pks, domain = setup
    wires, subnets, expect, root_a = _scenario(cur, domain)
    r = M.validate(wires, subnets, cur, N_VAL, lambda v: pks[v], SLOT, domain)
    return wires, subnets, expect, root_a, r


def test_statuses_and_roots(run):
    wires, subnets, expect, root_a, r = run
    assert r.status == expect
    assert r.roots == [root_a, ROOT_B]
    assert [r.root_id[a] for a in range(len(wires)) if expect[a] == M.ACCEPT] == [0] * 23 + [1] * 8
    assert all(r.root_id[a] == M.NONE for a in range(len(wires)) if expect[a] != M.ACCEPT)


def test_contributions_verify_over_their_subnet(setup, run):
    spec, state, cur, pks, domain = setup
    wires, subnets, expect, root_a, r = run
    assert sorted(r.contributions) == [(0, 0), (0, 1), (0, 2), (1, 3)]
    for (k, s), c in r.contributions.items():
        keys = [pks[cur[8 * s + i]] for i, b in enumerate(c.aggregation_bits) if b]
        assert eth_fast_aggregate_verify(keys, M.signing_root(r.roots[k], domain), c.signature)
        assert c.slot == SLOT and c.subcommittee_index == s and c.beacon_block_root == r.roots[k]
    # validator 3 holds positions 1 and 2: both bits, its signature twice in the sum
    c0 = r.contributions[(0, 0)]
    assert c0.aggregation_bits[1] and c0.aggregation_bits[2]
    sig3 = wires[[a for a in range(len(wires)) if expect[a] == M.ACCEPT and int.from_bytes(wires[a][40:48], "little") == 3][0]][48:144]
    others = [wires[a][48:144] for a in range(len(wires)) if expect[a] == M.ACCEPT and subnets[a] == 0 and r.root_id[a] == 0
              and int.from_bytes(wires[a][40:48], "little") != 3]
    assert c0.signature == B.Aggregate(others + [sig3, sig3])
    # the validator at positions 12 and 20 sent one message per subnet: each contribution carries its own bit
    assert r.contributions[(0, 1)].aggregation_bits[4] and r.contributions[(0, 2)].aggregation_bits[4]


def test_aggregates_pass_process_sync_aggregate(setup, run):
    spec, state, cur, pks, domain = setup
    wires, subnets, expect, root_a, r = run
    assert r.aggregates[0].sync_committee_bits == [p < 24 for p in range(32)]
    assert r.aggregates[1].sync_committee_bits == [p >= 24 for p in range(32)]
    for k, root in enumerate(r.roots):
        nxt = copy.deepcopy(state)
        nxt.slot = SLOT + 1
        nxt.block_roots[SLOT % len(nxt.block_roots)] = root
        before = list(nxt.balances)
        spec.process_sync_aggregate(nxt, r.aggregates[k])      # asserts eth_fast_aggregate_verify
        assert nxt.balances != before
        present = [r.contributions[(k, s)] for s in range(4) if (k, s) in r.contributions]
        assert r.aggregates[k] == M.process_sync_committee_contributions(present, 32)


def test_closed_form_sums(setup, run):
    spec, state, cur, pks, domain = setup
    wires, subnets, expect, root_a, r = run
    verdicts = {a: expect[a] != M.BAD_SIGNATURE for a in range(len(wires))}
    c = M.validate(wires, subnets, cur, N_VAL, lambda v: pks[v], SLOT, domain, verify=lambda a, pk, m, s: verdicts[a],
                   secret_key=scenarios.secret_key)
    assert c.status == r.status and c.roots == r.roots
    assert {k: x.signature for k, x in c.contributions.items()} == {k: x.signature for k, x in r.contributions.items()}
    assert [x.sync_committee_signature for x in c.aggregates] == [x.sync_committee_signature for x in r.aggregates]


def test_no_contribution_gives_the_infinity_aggregate():
    agg = M.process_sync_committee_contributions([], 32)
    assert agg.sync_committee_bits == [False] * 32 and agg.sync_committee_signature == M.G2_POINT_AT_INFINITY
    assert eth_fast_aggregate_verify([], bytes(32), agg.sync_committee_signature)


def test_serializer_matches_the_oracle():
    m = PS.SyncCommitteeMessage(123456789, ROOT_B, 4242, bytes(range(96)))
    w = PS.serialize_sync_committee_message(m)
    assert len(w) == M.WIRE and w == M.encode(123456789, ROOT_B, 4242, bytes(range(96)))
    assert PS.MINIMAL.SYNC_COMMITTEE_SUBNET_COUNT == PS.MAINNET.SYNC_COMMITTEE_SUBNET_COUNT == 4


# ------------------------------------------------------------------------------------------ the facade, with a stub engine
class _StubEngine:
    def __init__(self):
        self.calls = []

    def sync_committee_messages(self, wire, woff, subnet, position_validator, count, current_slot, domain32):
        n = len(woff) - 1
        self.calls.append((bytes(wire), list(woff), list(subnet), list(position_validator), count, current_slot, domain32))
        cb = np.zeros((1, count, 1), np.uint8)
        cb[0, 1, 0] = 0b101
        cs = np.zeros((1, count, 96), np.uint8)
        cs[0, 1] = 7
        ab = np.zeros((1, 4), np.uint8)
        ab[0, 1] = 0b101
        return SyncMessagesResult(np.arange(n, dtype=np.int32), np.zeros(n, np.uint32), np.full((1, 32), 9, np.uint8), cb, cs,
                                  np.array([[0, 1, 0, 0]], np.uint8), ab, np.full((1, 96), 8, np.uint8))


def _facade_state(slot):
    pks = [bytes([i]) * 48 for i in range(40)]
    cur = SyncCommittee([pks[(3 * i) % 40] for i in range(32)], bytes(48))
    nxt = SyncCommittee([pks[(7 * i + 1) % 40] for i in range(32)], bytes(48))
    return type("State", (), {"slot": slot, "validators": [PS.Validator(pk, 32 * 10**9) for pk in pks], "current_sync_committee": cur,
                              "next_sync_committee": nxt})(), cur, nxt


@pytest.mark.parametrize("slot,which", [(62, "current"), (63, "next"), (64, "current"), (127, "next")])
def test_facade_committee_choice(monkeypatch, slot, which):
    stub = _StubEngine()
    sp = PS.Spec(PS.MINIMAL, engine=stub)
    monkeypatch.setattr(sp, "sync_registry", lambda state: None)
    monkeypatch.setattr(sp, "get_domain", lambda state, d, epoch: bytes(d) + epoch.to_bytes(28, "little"))
    state, cur, nxt = _facade_state(slot)
    committee = cur if which == "current" else nxt
    msgs = [(1, PS.SyncCommitteeMessage(slot, bytes(32), 5, bytes(96))), (2**40, PS.SyncCommitteeMessage(slot, bytes(32), 6, bytes(95)))]
    status, contributions, aggregates = sp.validate_sync_committee_messages(state, msgs)
    wire, woff, subnet, pv, count, current_slot, domain = stub.calls[0]
    assert pv == [int(committee.pubkeys[p][0]) for p in range(32)]      # key i is validator i's
    assert count == 4 and current_slot == slot and domain == PS.DOMAIN_SYNC_COMMITTEE + (slot // 8).to_bytes(28, "little")
    assert woff == [0, 144, 287] and subnet == [1, 2**32 - 1] and wire[:144] == PS.serialize_sync_committee_message(msgs[0][1])
    assert status == [0, 1]
    assert contributions == [PS.SyncCommitteeContribution(slot, bytes([9]) * 32, 1, [True, False, True] + [False] * 5, bytes([7]) * 96)]
    agg = aggregates[bytes([9]) * 32]
    assert agg.sync_committee_bits == [i in (8, 10) for i in range(32)] and agg.sync_committee_signature == bytes([8]) * 96
    empty = aggregates[bytes(32)]
    assert bytes(32) not in aggregates and empty.sync_committee_bits == [False] * 32
    assert empty.sync_committee_signature == PS.G2_POINT_AT_INFINITY
    assert sp.validate_sync_committee_messages(state, []) == ([], [], {})


def test_facade_refuses_a_committee_key_outside_the_registry(monkeypatch):
    sp = PS.Spec(PS.MINIMAL, engine=_StubEngine())
    monkeypatch.setattr(sp, "sync_registry", lambda state: None)
    monkeypatch.setattr(sp, "get_domain", lambda state, d, epoch: bytes(32))
    state, cur, nxt = _facade_state(10)
    cur.pubkeys[3] = b"\xee" * 48
    with pytest.raises(ValueError):
        sp.validate_sync_committee_messages(state, [(0, PS.SyncCommitteeMessage(10, bytes(32), 5, bytes(96)))])
