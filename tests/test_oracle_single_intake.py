"""CPU checks of tests/single_intake_oracle.py: every status 0-13 at the minimal and mainnet committee counts per slot (M = 4 and 64),
the subnet rule on both sides of each committee's subnet, agreement with a pyspec-shaped restatement of the upstream Electra
beacon_attestation_{subnet_id} conditions and validate_on_attestation over oracle.spec with real signatures (the oracle's vote messages
are what the attesters signed), and equivalence with the phase 0 oracle on the same items written as phase 0 Attestations."""
import hashlib
import types

import numpy as np
import pytest

import intake_oracle as IO
import scenarios
import single_intake_oracle as SO
from oracle import bls_sig as B
from oracle import spec as S
from oracle.ssz import compute_domain

DOMAIN = compute_domain(bytes.fromhex("01000000"), bytes(4), bytes(32))
EPOCH = 3


def _tree(spe, seed=1, n_blocks=40):
    """a fork tree whose slots increase with the id; block 6 sits at start_slot(EPOCH)"""
    rng = np.random.default_rng(seed)
    parent = np.array([0] + [max(0, b - 1 - int(rng.integers(0, 3))) for b in range(1, n_blocks)], dtype=np.uint32)
    slot = (EPOCH * spe - 6 + np.arange(n_blocks)).astype(np.uint64)
    roots = np.frombuffer(b"".join(hashlib.sha256(b"single-block%d/%d" % (seed, b)).digest() for b in range(n_blocks)),
                          dtype=np.uint8).reshape(n_blocks, 32).copy()
    return parent, slot, roots


def _committees(n_c, size, seed=5):
    members = np.random.default_rng(seed).permutation(n_c * size).astype(np.uint32)
    return members, (np.arange(n_c + 1) * size).astype(np.uint32)


def every_status_case(tree, spe, cps, members, off):
    """(wires, subnets, current_slot): one or more items for each status 0-13 (the comment names it)"""
    parent, slot, roots = tree
    start = EPOCH * spe
    R = lambda b: bytes(roots[b])      # noqa: E731
    anc = lambda b: IO.ancestor(parent, slot, b, start)      # noqa: E731
    heads = [b for b in range(len(parent)) if int(slot[b]) <= start + 3 and anc(b) is not None]
    h1, h2 = heads[-1], heads[-2]
    ci = cps - 1                                                      # the slot's last committee: subnet (3 * cps + cps - 1) % 64
    c = 3 * cps + ci
    net = SO.compute_subnet_for_attestation(cps, start + 3, ci, spe, 64)
    mem = lambda p, cc=c: int(members[int(off[cc]) + p])      # noqa: E731

    def data(head, target=None, slot_=start + 3, index=0, tepoch=EPOCH):
        return IO.data128(slot_, index, R(head), EPOCH - 1, R(0), tepoch, R(anc(head)) if target is None else target)

    sig = lambda k: hashlib.sha256(b"sig%d" % k).digest() * 3      # noqa: E731
    A, Bd = data(h1), data(h2)
    items = [
        (SO.encode(ci, mem(0), A, sig(0)), net),                              # 0
        (SO.encode(ci, mem(1), Bd, sig(1)), net),                             # 0, another vote
        (SO.encode(ci, mem(2), A, sig(2)), net),                              # 0, the first vote again
        (SO.encode(ci, mem(0), A, sig(3)), net),                              # 13: duplicate, equal data
        (SO.encode(ci, mem(1), A, sig(4)), net),                              # 13: duplicate, other data
        (SO.encode(ci, mem(3), data(h1, target=R(0)), sig(5)), net),          # 12: target not the ancestor
        (SO.encode(ci, mem(3), A, sig(6)), net),                              # 0: the earlier item of this attester failed
        (SO.encode(ci, mem(4), A, sig(7))[:239], net),                        # 1: short
        (SO.encode(ci, mem(4), A, sig(7)) + b"\x00", net),                    # 1: long
        (b"", net),                                                           # 1: empty
        (SO.encode(ci, mem(4), data(h1, index=1), sig(8)), net),              # 2: data.index != 0
        (SO.encode(ci, mem(4), data(h1, index=ci), sig(8)), net),             # 2 (0 only at ci = 0: not this committee)
        (SO.encode(cps, mem(4), A, sig(9)), net),                             # 3: committee index = cps
        (SO.encode(2**64 - 1, mem(4), A, sig(9)), net),                       # 3
        (SO.encode(ci, mem(4), data(h1, slot_=start + spe), sig(10)), net),   # 4: the next epoch
        (SO.encode(ci, mem(4), data(h1, slot_=start - 1), sig(10)), net),     # 4: the epoch before
        (SO.encode(ci, mem(4), A, sig(11)), (net + 1) % 64),                  # 5: the next subnet
        (SO.encode(ci, mem(4), A, sig(11)), (net + 63) % 64),                 # 5: the one before
        (SO.encode(ci, mem(4), A, sig(11)), net + 64),                        # 5: not reduced mod 64
        (SO.encode(ci, mem(4), data(h1, tepoch=EPOCH + 1), sig(12)), net),    # 6: target epoch
        (SO.encode(ci, mem(4), data(h1, slot_=start + 7, target=R(anc(h1))),      # 7: current slot start + 7
                   sig(13)), SO.compute_subnet_for_attestation(cps, start + 7, ci, spe, 64)),
        (SO.encode(ci, mem(0, c - 1), A, sig(14)), net),                      # 8: a member of the committee before
        (SO.encode(ci, 10**9, A, sig(14)), net),                              # 8: no validator
        (SO.encode(ci, mem(4) + 2**32, A, sig(14)), net),                     # 8: the member's index plus 2^32
        (SO.encode(ci, mem(4), A[:16] + bytes([7] * 32) + A[48:], sig(15)), net),      # 9: unknown head
        (SO.encode(ci, mem(4), data(h1, target=bytes([9] * 32)), sig(16)), net),     # 10: unknown target
    ]
    newer = next(b for b in range(len(parent)) if int(slot[b]) > start + 3 and anc(b) is not None)
    items.append((SO.encode(ci, mem(4), data(newer), sig(17)), net))                 # 11: head newer than data.slot
    items.append((SO.encode(0, mem(0, 0), IO.data128(start, 0, R(heads[0]), EPOCH - 1, R(0), EPOCH, R(anc(heads[0]))), sig(18)),
                  SO.compute_subnet_for_attestation(cps, start, 0, spe, 64)))      # 0 in committee 0
    wires, subnets = zip(*items)
    return list(wires), np.array(subnets, dtype=np.uint32), start + 7


PRESETS = [(S.MINIMAL.SLOTS_PER_EPOCH, S.MINIMAL.MAX_COMMITTEES_PER_SLOT, 5), (S.MAINNET.SLOTS_PER_EPOCH, S.MAINNET.MAX_COMMITTEES_PER_SLOT, 5)]


@pytest.mark.parametrize("spe,cps,size", PRESETS, ids=["minimal", "mainnet"])
def test_every_status(spe, cps, size):
    tree = _tree(spe)
    members, off = _committees(spe * cps, size)
    wires, subnets, cur = every_status_case(tree, spe, cps, members, off)
    blocks, ids = IO.block_store(*tree)
    r = SO.single_intake_plain(wires, subnets, members, off, EPOCH, cur, DOMAIN, cps, spe, blocks, ids)
    want = [0, 0, 0, 13, 13, 12, 0, 1, 1, 1, 2, 2 if cps > 1 else 0, 3, 3, 4, 4, 5, 5, 5, 6, 7, 8, 8, 8, 9, 10, 11, 0]
    assert r.status.tolist() == want
    assert set(r.status.tolist()) == set(range(14))
    # the votes: committee (slot 3, cps - 1) has two, in the order of their smallest position; the other kept item is its committee's one
    c = 3 * cps + cps - 1
    assert int(r.vote_off[c + 1] - r.vote_off[c]) == 2
    row = r.vote[int(off[c]):int(off[c + 1])]
    assert row.tolist() == [int(r.vote_off[c]), int(r.vote_off[c]) + 1, int(r.vote_off[c]), int(r.vote_off[c]), SO.NONE]
    assert not r.data128[:, 8:16].any()                          # data as signed: data.index == 0
    assert int(r.vote_off[-1]) == spe * cps + 1


@pytest.mark.parametrize("spe,cps", [(8, 4), (32, 64)], ids=["minimal", "mainnet"])
def test_subnet_rule_at_every_committee(spe, cps):
    """each committee's items are kept on its own subnet only; the subnets of an epoch's committees cycle through all 64"""
    tree = _tree(spe)
    members, off = _committees(spe * cps, 1)
    parent, slot, roots = tree
    start = EPOCH * spe
    blocks, ids = IO.block_store(*tree)
    wires, subnets, want = [], [], []
    for c in range(spe * cps):
        s, ci = start + c // cps, c % cps
        b = int(np.nonzero(slot <= min(s, start))[0][-1])
        d = IO.data128(s, 0, bytes(roots[b]), EPOCH - 1, bytes(roots[0]), EPOCH, bytes(roots[IO.ancestor(parent, slot, b, start)]))
        net = (cps * (s % spe) + ci) % 64                        # the upstream formula, written out
        for k in (net, (net + 1) % 64):
            wires.append(SO.encode(ci, int(members[c]), d, bytes(96)))
            subnets.append(k)
            want.append(0 if k == net else 5)
    r = SO.single_intake_plain(wires, np.array(subnets), members, off, EPOCH, start + spe, DOMAIN, cps, spe, blocks, ids)
    assert r.status.tolist() == want
    assert sorted(set(subnets[0::2])) == list(range(min(64, spe * cps)))


def _pyspec_verdicts(spec, state, store, atts, subnet_ids, current_slot):
    """The upstream Electra beacon_attestation_{subnet_id} conditions in their order, then validate_on_attestation, over oracle.spec: True
    for an item a node accepts (REJECT and IGNORE both False).  Items arrive in list order at a node whose seen-cache is empty."""
    seen, out = set(), []
    for att, subnet_id in zip(atts, subnet_ids):
        data = att.data
        epoch = spec.compute_epoch_at_slot(data.slot)
        committees_per_slot = spec.get_committee_count_per_slot(state, epoch)
        ok = (data.index == 0                                                                  # [REJECT] Electra: data.index == 0
              and att.committee_index < committees_per_slot                                    # [REJECT] the committee index is in range
              and SO.compute_subnet_for_attestation(committees_per_slot, data.slot, att.committee_index, spec.p.SLOTS_PER_EPOCH, 64)
              == subnet_id                                                                     # [REJECT] the correct subnet
              and data.target.epoch == epoch                                                   # [REJECT] target epoch of the slot
              and epoch == EPOCH)                                                              # (this call's epoch)
        if ok:
            committee = spec.get_beacon_committee(state, data.slot, att.committee_index)
            ok = att.attester_index in committee                                               # [REJECT] the attester is a member
        if ok:
            ok = (att.attester_index, data.target.epoch) not in seen                           # [IGNORE] the first valid one of this attester
        if ok:
            indexed = S.IndexedAttestation([att.attester_index], data, att.signature)
            ok = spec.is_valid_indexed_attestation(state, indexed)                             # [REJECT] the signature
        if ok:                                                                                 # validate_on_attestation
            ok = (current_slot >= data.slot + 1 and data.beacon_block_root in store.blocks and data.target.root in store.blocks
                  and store.blocks[data.beacon_block_root].slot <= data.slot)
            if ok:
                try:
                    ok = spec.get_ancestor(store, data.beacon_block_root, spec.compute_start_slot_at_epoch(data.target.epoch)) == data.target.root
                except KeyError:
                    ok = False
        if ok:
            seen.add((att.attester_index, data.target.epoch))
        out.append(ok)
    return out


def test_matches_pyspec_rules_with_real_signatures():
    """Real signatures over the Electra data (index 0) by committee members of a minimal state: the oracle keeps exactly what the
    pyspec-shaped rules accept, and each of its votes' aggregates passes FastAggregateVerify over the voters' keys and its message."""
    from pos_evolution_b200.spec import AttestationData, Checkpoint, SingleAttestation, serialize_single_attestation
    spec, state = scenarios.minimal_state(64, slot=EPOCH * 8 + 5)
    spe = spec.p.SLOTS_PER_EPOCH
    cps = spec.get_committee_count_per_slot(state, EPOCH)
    start = EPOCH * spe
    parent, slot, roots = _tree(spe, seed=4)
    blocks, ids = IO.block_store(parent, slot, roots)
    store = types.SimpleNamespace(blocks=blocks)
    committees = [spec.get_beacon_committee(state, start + c // cps, c % cps) for c in range(spe * cps)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in committees])]).astype(np.uint32)
    members = np.array([v for x in committees for v in x], dtype=np.uint32)
    domain = spec.get_domain(state, S.DOMAIN_BEACON_ATTESTER, EPOCH)
    anc = lambda b: IO.ancestor(parent, slot, b, start)      # noqa: E731
    heads = [b for b in range(len(parent)) if int(slot[b]) <= start + 1 and anc(b) is not None]
    atts, nets = [], []
    for k, (c, p, h, tweak) in enumerate([(2, 0, heads[-1], None), (2, 1, heads[-2], None), (2, 2, heads[-1], None), (2, 0, heads[-2], None),
                                          (3, 0, heads[-1], "subnet"), (3, 1, heads[-1], "outsider"), (3, 2, heads[-1], "index"),
                                          (2, 3, heads[-1], "target"), (3, 3, heads[-1], None)]):
        s, ci = start + c // cps, c % cps
        who = int(committees[c][p]) if tweak != "outsider" else int(committees[c - 1][0])
        d = AttestationData(s, 1 if tweak == "index" else 0, bytes(roots[h]), Checkpoint(EPOCH - 1, bytes(roots[0])),
                            Checkpoint(EPOCH, bytes(roots[0]) if tweak == "target" else bytes(roots[anc(h)])))
        msg = S.Spec.compute_signing_root(S.AttestationData(d.slot, d.index, d.beacon_block_root, S.Checkpoint(d.source.epoch, d.source.root),
                                                            S.Checkpoint(d.target.epoch, d.target.root)), domain)
        atts.append(SingleAttestation(ci, who, d, scenarios.individual_signatures([who], msg)[0]))
        nets.append(SO.compute_subnet_for_attestation(cps, s, ci, spe, 64) + (1 if tweak == "subnet" else 0))
    wires = [serialize_single_attestation(a) for a in atts]
    r = SO.single_intake_plain(wires, nets, members, off, EPOCH, start + spe, domain, cps, spe, blocks, ids)
    spec_atts = [types.SimpleNamespace(committee_index=a.committee_index, attester_index=a.attester_index, signature=a.signature,
                                       data=S.AttestationData(a.data.slot, a.data.index, a.data.beacon_block_root,
                                                              S.Checkpoint(a.data.source.epoch, a.data.source.root),
                                                              S.Checkpoint(a.data.target.epoch, a.data.target.root))) for a in atts]
    verdicts = _pyspec_verdicts(spec, state, store, spec_atts, nets, start + spe)
    assert (r.status == 0).tolist() == verdicts
    assert r.status.tolist() == [0, 0, 0, 13, 5, 8, 2, 12, 0]
    for v in range(int(r.vote_off[-1])):
        pos = np.nonzero(r.vote == v)[0]
        if len(pos):
            agg = B.Aggregate([bytes(r.sigs[j]) for j in pos])
            assert B.FastAggregateVerify([state.validators[int(members[j])].pubkey for j in pos], bytes(r.msgs[v]), agg), v


@pytest.mark.parametrize("seed", range(3))
def test_equivalent_to_phase0_oracle(seed):
    """Each item that passes checks 1-8, written as the phase 0 Attestation with data.index = committee_index and one bit at the
    attester's position, gets the same status 0 or 9-13 from the phase 0 oracle, and the two give equal vote, vote_off, sigs, epochs and
    block ids; data128 differs only in bytes 8-15 and msgs in what that changes."""
    spe, cps, size = 8, 2, 5
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, 50, EPOCH * spe - 7)
    members, off = _committees(spe * cps, size, seed=seed)
    wires, subnets = SO.random_epoch(rng, EPOCH, spe, cps, members, off, tree, len(members), corrupt=0.4, dup=0.2, heads_per_committee=3)
    blocks, ids = IO.block_store(*tree)
    cur = (EPOCH + 1) * spe + 1
    r = SO.single_intake_plain(wires, subnets, members, off, EPOCH, cur, DOMAIN, cps, spe, blocks, ids)
    assert {0, 1, 8, 13} <= set(r.status.tolist()) and len(set(r.status.tolist())) >= 9
    passed = [i for i, s in enumerate(r.status.tolist()) if s == 0 or s >= 9]
    p0 = IO.intake_plain([SO.as_phase0(wires[i], members, off, cps, spe, EPOCH) for i in passed], off, EPOCH, cur, DOMAIN, cps, spe,
                         (size + 7) // 8, blocks, ids)
    assert p0.status.tolist() == r.status[passed].tolist()
    for f in ("vote", "vote_off", "sigs", "source_epoch", "target_epoch", "block_idx"):
        assert np.array_equal(getattr(p0, f), getattr(r, f)), f
    diff = p0.data128 != r.data128
    assert not diff[:, :8].any() and not diff[:, 16:].any()
