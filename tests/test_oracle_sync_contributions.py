"""Sync committee contributions on the CPU: tests/sync_contributions_oracle.py with real signatures on the minimal preset, against the
upstream rules it restates -- its roots against oracle/ssz.py's merkleize written out leaf by leaf, the product's serialiser against its
encoder, every accepted contribution through eth_fast_aggregate_verify over its subnet, every SyncAggregate through process_sync_aggregate
on the next slot's state, and the list-order cases of checks 8 and 9 and the choice of `best`."""
import copy

import pytest

import scenarios
import sync_contributions_oracle as C
from oracle.ssz import merkleize, sha256, uint_chunk
from pos_evolution_b200 import spec as PS
from sync_oracle import SyncCommittee, eth_aggregate_pubkeys, eth_fast_aggregate_verify, minimal_sync_state

N_VAL, SLOT = 64, 9
ROOT_A = scenarios._h(b"b200pos/blockroot" + SLOT.to_bytes(8, "little"))      # the state's block root at SLOT
ROOT_B = bytes(range(32))


def test_roots_against_merkleize():
    sig, proof = bytes(range(96)), bytes(range(96, 192))
    row = bytes([0x5A])
    z = bytes(32)
    sig_leaf = sha256(sha256(sig[:64]) + sha256(sig[64:] + z))
    assert C.sig_root(sig) == sig_leaf
    leaves = [uint_chunk(7), ROOT_B, uint_chunk(2), row + bytes(31), sig_leaf, z, z, z]
    assert C.contribution_root(7, ROOT_B, 2, row, sig) == merkleize(leaves)
    assert C.contribution_and_proof_root(5, 7, ROOT_B, 2, row, sig, proof) == \
        merkleize([uint_chunk(5), merkleize(leaves), C.sig_root(proof), z])
    assert C.selection_data_root(7, 2) == sha256(uint_chunk(7) + uint_chunk(2))
    # Bitvector[sub]: one chunk is the chunk itself; 2, 3 and 4 chunks pad to a power of two
    assert C.bitvector_root(bytes([1] * 16)) == bytes([1] * 16) + bytes(16)
    r128 = bytes(range(128))
    assert C.bitvector_root(r128) == merkleize([r128[0:32], r128[32:64], r128[64:96], r128[96:128]])
    assert C.bitvector_root(r128[:80]) == merkleize([r128[0:32], r128[32:64], r128[64:80] + bytes(16), z])
    assert C.bitvector_root(r128[:40]) == sha256(r128[0:32] + r128[32:40] + bytes(24))


def test_product_serialiser_matches_encoder():
    bits = [bool(i % 3 == 0) for i in range(8)]
    c = PS.SyncCommitteeContribution(11, ROOT_B, 3, bits, bytes([1]) * 96)
    s = PS.SignedContributionAndProof(PS.ContributionAndProof(42, c, bytes([2]) * 96), bytes([3]) * 96)
    w = PS.serialize_signed_contribution_and_proof(s)
    assert len(w) == 345 and w == C.encode(42, 11, ROOT_B, 3, bits, bytes([1]) * 96, bytes([2]) * 96, bytes([3]) * 96)
    assert PS.MINIMAL.TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE == 16
    assert PS.DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF == bytes([8, 0, 0, 0]) and PS.DOMAIN_CONTRIBUTION_AND_PROOF == bytes([9, 0, 0, 0])


def test_malformed_bitvector_and_length():
    pv = list(range(12))      # committee 12 over 4 subnets: Bitvector[3], one byte with five unused bits
    ok = C.encode(1, SLOT, ROOT_B, 0, [True, False, True], bytes(96), bytes(96), bytes(96))
    high = bytearray(ok)
    high[56] |= 0x08
    r = C.validate([ok[:-1], bytes(high), ok + b"\0"], pv, N_VAL, None, SLOT, bytes(96), target=16)
    assert r.status == [C.MALFORMED] * 3


@pytest.fixture(scope="module")
def setup():
    pks = scenarios.pubkeys(N_VAL)
    spec, state, cur = minimal_sync_state(N_VAL, slot=SLOT, pks=pks)
    epoch = spec.compute_epoch_at_slot(SLOT)
    domains = b"".join(spec.get_domain(state, d, epoch) for d in (PS.DOMAIN_SYNC_COMMITTEE, PS.DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF,
                                                                  PS.DOMAIN_CONTRIBUTION_AND_PROOF))
    pv = C.with_aggregators(cur, N_VAL, lambda p: C.Signer(p, domains, SLOT), 1, {1: 2, 2: 2, 3: 1})
    state.current_sync_committee = SyncCommittee([pks[v] for v in pv], eth_aggregate_pubkeys([pks[v] for v in pv]))
    return spec, state, pv, pks, domains


def test_every_status_with_real_signatures(setup):
    spec, state, pv, pks, domains = setup
    sg = C.Signer(pv, domains, SLOT)
    wires, expect = C.scenario(sg, [ROOT_A, ROOT_B], 1, N_VAL)
    r = C.validate(wires, pv, N_VAL, lambda v: pks[v], SLOT, domains, target=1)
    assert r.status == expect and set(expect) == set(range(13))
    assert r.roots == [ROOT_A, ROOT_B]
    # best: a1's on (A, 1); a3's on (B, 1); b1's and b2's two-bit contributions tie on (B, 2): the smaller index wins
    acc = [a for a, st in enumerate(r.status) if st == C.ACCEPT]
    assert r.best[0] == [C.NONE, acc[0], C.NONE, C.NONE] and r.best[1] == [C.NONE, acc[1], acc[2], C.NONE]
    sub = len(pv) // C.SUBNET_COUNT
    for a in acc:      # every accepted contribution verifies over its subnet's keys, a key counted once per set position
        g, slot, root, s, row, sig, _, _ = C.decode(wires[a], 1)
        keys = [pks[pv[s * sub + i]] for i in range(sub) if row[0] >> i & 1]
        assert eth_fast_aggregate_verify(keys, C.signing_root(root, domains[:32]), sig)
    for k, root in enumerate(r.roots):
        nxt = copy.deepcopy(state)
        nxt.slot = SLOT + 1
        nxt.block_roots[SLOT % len(nxt.block_roots)] = root
        spec.process_sync_aggregate(nxt, r.aggregates[k])


def test_list_order_cases(setup):
    """the scenario's cases one by one, each against the statuses the rules give"""
    spec, state, pv, pks, domains = setup
    sg = C.Signer(pv, domains, SLOT)
    sub = sg.sub
    a1, b1 = pv[sub], pv[2 * sub]
    on = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    run = lambda ws: C.validate(ws, pv, N_VAL, lambda v: pks[v], SLOT, domains, target=16).status      # noqa: E731
    x = sg.item(a1, 1, ROOT_A, on(0, 1, 2))
    assert run([x, x]) == [C.ACCEPT, C.COVERED]                                         # an equal-bits duplicate
    sup_bad = sg.item(a1, 1, ROOT_A, on(0, 1, 2, 3), bad_sig=True)
    assert run([sup_bad, x]) == [C.BAD_CONTRIBUTION, C.ACCEPT]                          # a subset after a rejected superset
    assert run([x, sg.item(a1, 1, ROOT_B, on(5))]) == [C.ACCEPT, C.SEEN_AGGREGATOR]     # the same aggregator on a second root
    bad = sg.item(a1, 1, ROOT_A, on(0, 1, 2), proof=sg.bad_proof(a1, 1, 16))
    assert run([bad, x]) == [C.BAD_PROOF, C.ACCEPT]                                     # a bad selection proof shadows nothing
    y, z = sg.item(b1, 2, ROOT_A, on(1, 2)), sg.item(pv[2 * sub + 1], 2, ROOT_A, on(5, 6))
    r = C.validate([y, z], pv, N_VAL, lambda v: pks[v], SLOT, domains, target=16)
    assert r.status == [C.ACCEPT, C.ACCEPT] and r.best == [[C.NONE, C.NONE, 0, C.NONE]]   # ties go to the smaller list index
    r = C.validate([z, y], pv, N_VAL, lambda v: pks[v], SLOT, domains, target=16)
    assert r.best == [[C.NONE, C.NONE, 0, C.NONE]]
