"""tests/block_attestations_electra_oracle.py against a pyspec-shaped Electra process_attestation (Deneb's inclusion window and flags, EIP-7549
committee_bits), written here over oracle.spec objects and run block by block on the minimal preset (4-bit committee_bits, 2 committees per
slot at 64 validators), with real oracle.bls_sig signatures: every status 0-13, the Deneb windows, and block-atomic runs.  Also: one-committee
attestations inside the Altair window give block_attestations_oracle.run's flags, numerators and tables on their phase 0 encodings."""
import copy
import functools
import hashlib

import numpy as np
import pytest

import block_attestations_electra_oracle as E
import block_attestations_oracle as O
import scenarios
from oracle import bls_sig as B
from oracle import spec as S
from oracle.bls12_381 import R
from oracle.spec import PARTICIPATION_FLAG_WEIGHTS, PROPOSER_WEIGHT, WEIGHT_DENOMINATOR, integer_squareroot

SPE, M = S.MINIMAL.SLOTS_PER_EPOCH, S.MINIMAL.MAX_COMMITTEES_PER_SLOT        # 8, 4
MAX_VPC = S.MINIMAL.MAX_VALIDATORS_PER_COMMITTEE
PKS = scenarios.pubkeys(64)


def _h(b):
    return hashlib.sha256(b).digest()


@functools.lru_cache(maxsize=None)
def _fav(pubkeys, msg, sig):
    return B.FastAggregateVerify(list(pubkeys), msg, sig)


class RealBLS:
    @staticmethod
    def FastAggregateVerify(pubkeys, msg, sig):
        return _fav(tuple(bytes(p) for p in pubkeys), bytes(msg), bytes(sig))


class Att:
    """an Electra Attestation over oracle.spec's AttestationData"""

    def __init__(self, aggregation_bits, data, signature, committee_bits):
        self.aggregation_bits, self.data, self.signature, self.committee_bits = aggregation_bits, data, signature, committee_bits


def deneb_flag_indices(sp, state, data, inclusion_delay):
    """get_attestation_participation_flag_indices, Deneb (EIP-7045)"""
    justified = state.current_justified_checkpoint if data.target.epoch == sp.get_current_epoch(state) else state.previous_justified_checkpoint
    is_matching_source = data.source == justified
    is_matching_target = is_matching_source and data.target.root == sp.get_block_root(state, data.target.epoch)
    is_matching_head = is_matching_target and data.beacon_block_root == sp.get_block_root_at_slot(state, data.slot)
    assert is_matching_source
    flags = []
    if is_matching_source and inclusion_delay <= integer_squareroot(sp.p.SLOTS_PER_EPOCH):
        flags.append(0)
    if is_matching_target:
        flags.append(1)
    if is_matching_head and inclusion_delay == sp.p.MIN_ATTESTATION_INCLUSION_DELAY:
        flags.append(2)
    return flags


def electra_process_attestation(sp, state, att):
    """process_attestation of upstream Electra beacon-chain.md (with Deneb's window), over oracle.spec"""
    data = att.data
    assert data.target.epoch in (sp.get_previous_epoch(state), sp.get_current_epoch(state))
    assert data.target.epoch == sp.compute_epoch_at_slot(data.slot)
    assert data.slot + sp.p.MIN_ATTESTATION_INCLUSION_DELAY <= state.slot
    assert data.index == 0
    committee_indices = [i for i, b in enumerate(att.committee_bits) if b]
    committee_offset, attesting = 0, set()
    for committee_index in committee_indices:
        assert committee_index < sp.get_committee_count_per_slot(state, data.target.epoch)
        committee = sp.get_beacon_committee(state, data.slot, committee_index)
        try:
            committee_attesters = set(a for i, a in enumerate(committee) if att.aggregation_bits[committee_offset + i])
        except IndexError:
            raise AssertionError("read past the Bitlist")
        assert len(committee_attesters) > 0
        attesting |= committee_attesters
        committee_offset += len(committee)
    assert len(att.aggregation_bits) == committee_offset
    flag_indices = deneb_flag_indices(sp, state, data, state.slot - data.slot)
    assert sp.is_valid_indexed_attestation(state, S.IndexedAttestation(sorted(attesting), data, att.signature))
    cur = data.target.epoch == sp.get_current_epoch(state)
    participation = state.current_epoch_participation if cur else state.previous_epoch_participation
    numerator = 0
    for index in attesting:
        for flag_index, weight in enumerate(PARTICIPATION_FLAG_WEIGHTS):
            if flag_index in flag_indices and not sp.has_flag(participation[index], flag_index):
                participation[index] = sp.add_flag(participation[index], flag_index)
                numerator += sp.get_base_reward(state, index) * weight
    denominator = (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT) * WEIGHT_DENOMINATOR // PROPOSER_WEIGHT
    sp.increase_balance(state, sp.get_beacon_proposer_index(state), numerator // denominator)


class Run:
    """a run of blocks on a 64-validator minimal state at epoch 2; atts[k] holds Att objects or raw encodings"""

    def __init__(self, slots, first=None):
        self.slots = list(slots)
        _, st = scenarios.minimal_state(64, slot=self.slots[0] if first is None else first, pks=PKS)
        st.slot = self.slots[0]
        st.previous_justified_checkpoint = S.Checkpoint(1, _h(b"j1"))
        st.current_justified_checkpoint = S.Checkpoint(2, _h(b"j2"))
        self.spec, self.state = S.Spec(S.MINIMAL, bls_module=RealBLS), st
        self.H = S.MINIMAL.SLOTS_PER_HISTORICAL_ROOT
        self.roots = [_h(b"block" + s.to_bytes(8, "little")) for s in self.slots]
        self.atts = [[] for _ in self.slots]

    def root(self, s):
        if s < self.slots[0]:
            return bytes(self.state.block_roots[s % self.H])
        return [r for r, b in zip(self.roots, self.slots) if b <= s][-1]

    def make(self, slot, picks, bits=None, index=0, head=None, target_root=None, target_epoch=None, source=None, corrupt=False):
        sp, st = self.spec, self.state
        e = self.slots[0] // SPE
        tepoch = slot // SPE if target_epoch is None else target_epoch
        cps = sp.get_committee_count_per_slot(st, slot // SPE)
        rows = [sp.get_beacon_committee(st, slot, i) if i < cps else [0, 1, 2] for i in picks]
        flat = [v for r in rows for v in r]
        bits = [True] * len(flat) if bits is None else list(bits)
        if source is None:
            source = st.current_justified_checkpoint if tepoch == e else st.previous_justified_checkpoint
        data = S.AttestationData(slot, index, self.root(slot) if head is None else head, source,
                                 S.Checkpoint(tepoch, self.root(tepoch * SPE) if target_root is None else target_root))
        signers = sorted(set(v for v, b in zip(flat, bits) if b))
        msg = sp.compute_signing_root(data, sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, tepoch))
        sk = (sum(scenarios.secret_key(v) for v in signers) + (1 if corrupt else 0)) % R or 1
        return Att(bits, data, B.Sign(sk, msg), E.committee_bits_of(picks, M))

    @staticmethod
    def encode(a):
        d = a.data
        return E.encode(a.aggregation_bits, E.data128(d.slot, d.index, d.beacon_block_root, d.source.epoch, d.source.root, d.target.epoch,
                                                      d.target.root), a.signature, a.committee_bits)

    def inputs(self):
        sp, st = self.spec, self.state
        e = self.slots[0] // SPE
        members, off, cps = [], [0], []
        for Ep in (e - 1, e):
            cps.append(sp.get_committee_count_per_slot(st, Ep))
            for s in range(Ep * SPE, (Ep + 1) * SPE):
                for i in range(cps[-1]):
                    members += sp.get_beacon_committee(st, s, i)
                    off.append(len(members))
        wires = [[a if isinstance(a, bytes) else self.encode(a) for a in blk] for blk in self.atts]
        wire, woff, block_off = O.layout(wires)
        cp = lambda c: c.epoch.to_bytes(8, "little") + c.root      # noqa: E731
        return dict(wire=wire, woff=woff, block_off=block_off, block_slot=self.slots, members=np.array(members, np.uint32),
                    off=np.array(off, np.uint32), cps_prev=cps[0], cps_cur=cps[1],
                    chain_roots=[self.root(s) for s in range(e * SPE - SPE, e * SPE + SPE)],
                    justified80=cp(st.previous_justified_checkpoint) + cp(st.current_justified_checkpoint),
                    domains64=sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, e - 1) + sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, e), spe=SPE,
                    min_delay=1, eff=[v.effective_balance for v in st.validators], increment=sp.p.EFFECTIVE_BALANCE_INCREMENT,
                    per_increment=sp.get_base_reward_per_increment(st), part_cur=st.current_epoch_participation,
                    part_prev=st.previous_epoch_participation)

    def oracle(self):
        keys = [v.pubkey for v in self.state.validators]
        verify = lambda idx, root, sig: RealBLS.FastAggregateVerify([keys[v] for v in idx], root, sig)      # noqa: E731
        return E.run(M=M, max_vpc=MAX_VPC, verify=verify, **self.inputs())

    def spec_blocks(self):
        """(state after the run, the first block that raised or None, its failing attestation)"""
        st = copy.deepcopy(self.state)
        for k, s in enumerate(self.slots):
            if k:
                for t in range(self.slots[k - 1], s):
                    st.block_roots[t % self.H] = self.roots[k - 1]
            st.slot = s
            before = copy.deepcopy(st)
            for j, a in enumerate(self.atts[k]):
                try:
                    if isinstance(a, bytes):
                        raise AssertionError("does not decode")
                    electra_process_attestation(self.spec, st, a)
                except AssertionError:
                    return before, k, j
        return st, None, None

    def check(self):
        """the oracle against the spec block by block; returns the oracle's result"""
        r = self.oracle()
        st, k, j = self.spec_blocks()
        assert r["n_applied"] == (len(self.slots) if k is None else k)
        if k is not None:
            assert r["block_status"][k] == 1 and r["block_first"][k] == j
        assert r["part_cur"] == list(st.current_epoch_participation)
        assert r["part_prev"] == list(st.previous_epoch_participation)
        bal = list(self.state.balances)
        for b in range(r["n_applied"]):
            at = copy.copy(self.state)
            at.slot = self.slots[b]
            bal[self.spec.get_beacon_proposer_index(at)] += int(r["block_reward"][b])
        assert bal == list(st.balances)
        return r


def _bad(run, status, s):
    """an attestation for a block at slot s that fails with `status`"""
    F = E.fixed(M)
    good = Run.encode(run.make(s - 1, [0, 1]))
    if status == 1:
        return good[:F - 3]
    if status == 2:
        return good[:F]
    if status == 3:
        return good[:F] + E.bitlist([True] * (MAX_VPC * M + 1))
    return {4: lambda: run.make(2, [0], target_epoch=0), 5: lambda: run.make(s - 9, [0], target_epoch=2), 6: lambda: run.make(s, [0]),
            7: lambda: run.make(s - 1, [0], index=1), 8: lambda: run.make(s - 1, [0, 2]),
            9: lambda: run.make(s - 1, [0, 1], bits=[True] * 4 + [False] * 4),
            10: lambda: run.make(s - 1, [0, 1], bits=[True] * 7), 11: lambda: run.make(s - 1, [1], source=S.Checkpoint(1, _h(b"j1"))),
            12: lambda: run.make(s - 1, []), 13: lambda: run.make(s - 1, [1], corrupt=True)}[status]()


@pytest.mark.parametrize("status", range(1, 14))
def test_every_status_stops_the_run_at_its_block(status):
    run = Run([17, 19, 21])
    run.atts[0] = [run.make(16, [0, 1]), run.make(9, [1])]
    run.atts[1] = [run.make(18, [1]), _bad(run, status, 19)]
    run.atts[2] = [run.make(20, [0])]
    r = run.check()
    assert r["status"].tolist()[2:4] == [0, status] and r["n_applied"] == 1 and r["block_status"].tolist() == [0, 1, 2]


def test_deneb_windows_and_flags():
    """delays 1, 2 = isqrt(8), 3, 8, 9 and 15 (the previous epoch's first slot from the last slot of e): target past SLOTS_PER_EPOCH, head
    only at 1; a wrong head or target root; every committee of a slot in one aggregate; re-inclusions that earn nothing"""
    run = Run([21, 23])
    run.atts[0] = [run.make(20, [0, 1]), run.make(19, [0]), run.make(18, [1]), run.make(13, [0, 1]), run.make(12, [1]),
                   run.make(20, [1], head=_h(b"other")), run.make(19, [1], target_root=_h(b"t"))]
    run.atts[1] = [run.make(8, [0]), run.make(8, [1], bits=[True, False] * 2), run.make(20, [0, 1]), run.make(22, [0])]
    r = run.check()
    assert r["status"].tolist() == [0] * 11 and r["n_applied"] == 2
    assert r["flag_mask"].tolist() == [7, 3, 2, 2, 2, 3, 1, 2, 2, 2, 7]
    assert r["numerator"][9] == 0 and r["numerator"][0] > 0


def test_single_committee_matches_the_phase0_oracle():
    """one-committee Electra attestations within the Altair window: the flags, numerators and tables of block_attestations_oracle.run on
    their phase 0 encodings (data.index = the committee; the phase 0 run's index is that committee)"""
    run = Run([18, 20, 22])
    specs = [[(17, 0), (17, 1), (12, 1), (11, 0)], [(19, 1), (18, 0), (14, 0)], [(21, 0), (21, 1), (17, 0), (15, 1)]]
    electra, phase0 = [], []
    for blk in specs:
        e_blk, p_blk = [], []
        for slot, c in blk:
            a = run.make(slot, [c], bits=[(j + c) % 3 != 0 for j in range(4)])
            e_blk.append(a)
            d = a.data
            p_blk.append(O.encode(a.aggregation_bits, O.data128(d.slot, c, d.beacon_block_root, d.source.epoch, d.source.root, d.target.epoch,
                                                                d.target.root), a.signature))
        electra.append(e_blk)
        phase0.append(p_blk)
    run.atts = electra
    r = run.oracle()
    inp = run.inputs()
    wire, woff, block_off = O.layout(phase0)
    keys = [v.pubkey for v in run.state.validators]
    p0 = O.run(wire, woff, block_off, run.slots, inp["members"], inp["off"], inp["cps_prev"], inp["cps_cur"], inp["chain_roots"],
               inp["justified80"], inp["domains64"], SPE, 1, 1, inp["eff"], inp["increment"], inp["per_increment"], inp["part_cur"],
               inp["part_prev"], lambda idx, root, sig: True)
    assert r["status"].tolist() == [0] * 11 and p0["status"].tolist() == [0] * 11
    for k in ("flag_mask", "numerator", "block_reward"):
        assert r[k].tolist() == p0[k].tolist(), k
    assert r["part_cur"] == p0["part_cur"] and r["part_prev"] == p0["part_prev"]
