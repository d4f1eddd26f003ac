"""tests/block_attestations_oracle.py against oracle.spec.process_attestation run block by block (CPU): for each block the state's slot is
set, the skipped slots' block_roots are written, and the block's attestations are processed one by one; a block whose attestation raises
leaves the state as it was before it, and no later block is processed.  The comparison covers raise / no raise, the failing attestation,
both participation tables and the balances (each applied block's reward credited to get_beacon_proposer_index at its slot).  Signatures
are checked by a stand-in FastAggregateVerify (a hash of the keys and the message) that both sides share."""
import copy
import hashlib

import numpy as np
import pytest

import block_attestations_oracle as O
import scenarios
from oracle import spec as S

SPE = S.MINIMAL.SLOTS_PER_EPOCH          # 8; integer_squareroot = 2


def _h(b):
    return hashlib.sha256(b).digest()


def fake_sig(pubkeys, msg):
    return _h(b"".join(pubkeys) + msg) * 3


class FakeBLS:
    @staticmethod
    def FastAggregateVerify(pubkeys, msg, sig):
        return len(pubkeys) > 0 and bytes(sig) == fake_sig(pubkeys, msg)


PKS = [_h(b"pk" + i.to_bytes(4, "little")) + bytes(16) for i in range(64)]


def make_state(slot, late=0):
    """64 validators on the minimal preset; the last `late` of them become active at epoch 2 (fewer committees before it)"""
    _, st = scenarios.minimal_state(64, slot=slot, pks=PKS)
    for v in st.validators[64 - late:]:
        v.activation_epoch = 2
    st.previous_justified_checkpoint = S.Checkpoint(0, _h(b"j0"))
    st.current_justified_checkpoint = S.Checkpoint(1 if slot >= SPE else 0, _h(b"j1") if slot >= SPE else _h(b"j0"))
    return S.Spec(S.MINIMAL, bls_module=FakeBLS), st


class Run:
    """A run of blocks on a state: blocks[k] = (slot, root); roots(s) is the chain's block root at slot s as the last block sees it.  The
    epoch length and the block-root ring come from the spec's preset."""

    def __init__(self, spec, state, slots):
        self.spec, self.state, self.slots = spec, state, list(slots)
        self.spe, self.H = spec.p.SLOTS_PER_EPOCH, spec.p.SLOTS_PER_HISTORICAL_ROOT
        self.roots = [_h(b"block" + s.to_bytes(8, "little")) for s in self.slots]
        self.atts = [[] for _ in self.slots]

    def root(self, s):
        if s < self.slots[0]:
            return bytes(self.state.block_roots[s % self.H]) if s >= 0 else bytes(32)
        return [r for r, b in zip(self.roots, self.slots) if b <= s][-1]

    def add(self, k, slot, index, bits=None, head=None, target_root=None, target_epoch=None, source=None, bad_sig=False):
        """an attestation of (slot, index) in block k, right in every field unless one is given"""
        sp, st, SPE = self.spec, self.state, self.spe
        e = slot // SPE
        tepoch = e if target_epoch is None else target_epoch
        cur = self.slots[0] // SPE
        committee = sp.get_beacon_committee(st, slot, index) if index < sp.get_committee_count_per_slot(st, e) else [0] * 4
        bits = [True] * len(committee) if bits is None else list(bits)
        if source is None:
            source = st.current_justified_checkpoint if tepoch == cur else st.previous_justified_checkpoint
        data = S.AttestationData(slot, index, self.root(slot) if head is None else head, source,
                                 S.Checkpoint(tepoch, self.root(tepoch * SPE) if target_root is None else target_root))
        signers = sorted(set(v for v, b in zip(committee, bits) if b))
        msg = sp.compute_signing_root(data, sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, tepoch))
        sig = fake_sig([st.validators[v].pubkey for v in signers], msg)
        if bad_sig:
            sig = _h(sig) * 3
        self.atts[k].append(S.Attestation(bits, data, sig))

    def inputs(self):
        sp, st, SPE = self.spec, self.state, self.spe
        e = self.slots[0] // SPE
        members, off, cps = [], [0], []
        for E in ([e - 1] if e > 0 else []) + [e]:
            cps.append(sp.get_committee_count_per_slot(st, E))
            for s in range(E * SPE, (E + 1) * SPE):
                for i in range(cps[-1]):
                    members += sp.get_beacon_committee(st, s, i)
                    off.append(len(members))
        cps_prev, cps_cur = (cps[0], cps[1]) if e > 0 else (0, cps[0])
        wires = [[a if isinstance(a, bytes) else self.encode(a) for a in blk] for blk in self.atts]
        wire, woff, block_off = O.layout(wires)
        stride = max(1, (max(np.diff(off)) + 7) // 8)
        roots = [self.root(s) for s in range(e * SPE - SPE, e * SPE + SPE)]
        cp = lambda c: c.epoch.to_bytes(8, "little") + c.root      # noqa: E731
        justified = cp(st.previous_justified_checkpoint) + cp(st.current_justified_checkpoint)
        domains = sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, max(e, 1) - 1) + sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, e)
        return dict(wire=wire, woff=woff, block_off=block_off, block_slot=self.slots, members=np.array(members, np.uint32),
                    off=np.array(off, np.uint32), cps_prev=cps_prev, cps_cur=cps_cur, chain_roots=roots, justified80=justified,
                    domains64=domains, spe=SPE, min_delay=sp.p.MIN_ATTESTATION_INCLUSION_DELAY, bits_stride=stride,
                    eff=[v.effective_balance for v in st.validators], increment=sp.p.EFFECTIVE_BALANCE_INCREMENT,
                    per_increment=sp.get_base_reward_per_increment(st), part_cur=st.current_epoch_participation,
                    part_prev=st.previous_epoch_participation)

    @staticmethod
    def encode(a):
        d = a.data
        return O.encode(a.aggregation_bits, O.data128(d.slot, d.index, d.beacon_block_root, d.source.epoch, d.source.root, d.target.epoch,
                                                     d.target.root), a.signature)

    def oracle(self):
        keys = [v.pubkey for v in self.state.validators]
        verify = lambda idx, root, sig: bytes(sig) == fake_sig([keys[v] for v in idx], root)      # noqa: E731
        return O.run(verify=verify, **self.inputs())

    def proposers(self):
        out = []
        for s in self.slots:
            st = copy.copy(self.state)
            st.slot = s
            out.append(self.spec.get_beacon_proposer_index(st))
        return out

    def spec_blocks(self):
        """(state after the run, index of the first block that raised or None, its failing attestation)"""
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
                    self.spec.process_attestation(st, a)
                except AssertionError:
                    return before, k, j
        return st, None, None


def check(run):
    """the oracle against the spec block by block; returns the oracle's result"""
    r = run.oracle()
    st, k, j = run.spec_blocks()
    n = len(run.slots)
    assert r["n_applied"] == (n if k is None else k)
    if k is not None:
        assert r["block_status"][k] == 1 and r["block_first"][k] == j
    assert all(r["block_status"][b] == 0 for b in range(r["n_applied"]))
    assert r["part_cur"] == list(st.current_epoch_participation)
    assert r["part_prev"] == list(st.previous_epoch_participation)
    bal = list(run.state.balances)
    for b, p in zip(range(r["n_applied"]), run.proposers()):
        bal[p] += int(r["block_reward"][b])
    assert bal == list(st.balances)
    return r


def _epoch2_run(late=0, slots=(17, 19, 21)):
    spec, st = make_state(slots[0], late)
    return Run(spec, st, slots)


def _good(run, k):
    """two valid attestations into block k: one of each epoch"""
    s = run.slots[k]
    run.add(k, s - 1, 0)
    run.add(k, s - 6, 1)


MALFORMED = {1: lambda w: w[:200], 2: lambda w: w[:228]}     # a truncated container; an empty Bitlist


@pytest.mark.parametrize("status", range(1, 12))
def test_every_status_stops_the_run_at_its_block(status):
    run = _epoch2_run()
    _good(run, 0)
    _good(run, 1)
    s = run.slots[1]
    if status in (1, 2):
        run.add(1, s - 1, 1)
        run.atts[1][-1] = MALFORMED[status](Run.encode(run.atts[1][-1]))
    elif status == 3:
        run.add(1, s - 1, 1, bits=[True] * 9)
    elif status == 4:
        run.add(1, 2, 0, target_epoch=0)                      # target e - 2
    elif status == 5:
        run.add(1, s - 9, 0, target_epoch=2)                  # a slot of epoch 1 with target 2
    elif status == 6:
        run.add(1, s - 9, 0)                                  # inclusion delay SLOTS_PER_EPOCH + 1
    elif status == 7:
        run.add(1, s - 1, 2)
    elif status == 8:
        run.add(1, s - 1, 0, bits=[True] * 3)
    elif status == 9:
        run.add(1, s - 1, 0, source=S.Checkpoint(0, _h(b"j0")))    # the previous justified checkpoint for a current target
    elif status == 10:
        run.add(1, s - 1, 0, bits=[False] * 4)
    elif status == 11:
        run.add(1, s - 1, 0, bad_sig=True)
    _good(run, 1)
    _good(run, 2)
    r = check(run)
    assert r["status"][4] == status and r["block_first"][1] == 2 and r["n_applied"] == 1
    assert r["status"].tolist().count(0) == 8 and list(r["block_status"]) == [0, 1, 2]


def test_delay_boundaries_and_flag_masks():
    """inclusion delays 1, 2 = isqrt(8), 3, 8 in one block at the epoch's last slot, head and target mismatches; delay 9 is status 6"""
    run = _epoch2_run(slots=(23,))
    for delay in (1, 2, 3, 8):
        run.add(0, 23 - delay, 0)
    run.add(0, 22, 1, target_root=_h(b"other target"), head=_h(b"x"))
    run.add(0, 22, 1, head=_h(b"other head"))
    run.add(0, 14, 0)                                         # delay 9, in e - 1
    r = check(run)
    assert r["status"].tolist() == [0, 0, 0, 0, 0, 0, 6] and r["n_applied"] == 0
    assert r["flag_mask"].tolist()[:6] == [7, 3, 2, 2, 1, 3]
    run.atts[0].pop()
    r = check(run)
    assert r["n_applied"] == 1 and all(r["numerator"] > 0)


def test_overlapping_aggregates_earn_only_what_is_left():
    """the same committees across consecutive blocks: full, then subsets, then exact repeats; a later block earns only the remaining flags"""
    run = _epoch2_run(slots=(18, 19, 20, 22))
    run.add(0, 17, 0, bits=[True, False, True, False])
    run.add(0, 17, 0, bits=[True, True, False, False])
    run.add(1, 17, 0)
    run.add(1, 17, 0)
    run.add(2, 17, 0, bits=[False, False, False, True])
    run.add(2, 19, 1)
    run.add(3, 19, 1)
    run.add(3, 15, 0)
    run.add(3, 15, 0)
    r = check(run)
    assert r["n_applied"] == 4 and r["status"].tolist() == [0] * 9
    assert [int(x) > 0 for x in r["numerator"]] == [True, True, True, False, False, True, False, True, False]


def test_epoch_zero():
    spec, st = make_state(3)
    run = Run(spec, st, (3, 5, 7))
    run.add(0, 2, 0)
    run.add(0, 0, 1)
    run.add(1, 4, 1)
    run.add(1, 3, 0, bits=[False, True, True, False])
    run.add(2, 6, 0)
    run.add(2, 4, 0)
    r = check(run)
    assert r["n_applied"] == 3 and not any(r["part_prev"])
    run.add(2, 6, 1, target_epoch=1)                          # no previous epoch at 0: target 1 is neither
    r = check(run)
    assert r["status"][-1] == 4 and r["n_applied"] == 2
    run.atts[2].pop()
    run.add(2, 5, 1, target_epoch=0, head=_h(b"h"))
    assert check(run)["n_applied"] == 3


def test_committee_counts_differ_between_epochs():
    """32 validators join at epoch 2: one committee per slot in epoch 1, two in epoch 2"""
    run = _epoch2_run(late=32)
    assert run.inputs()["cps_prev"] == 1 and run.inputs()["cps_cur"] == 2
    run.add(0, 16, 1)
    run.add(0, 12, 0)
    run.add(1, 18, 0)
    run.add(1, 15, 0, bits=[True, False, True, True])
    run.add(2, 13, 1)                                          # index 1 of an epoch with one committee per slot
    r = check(run)
    assert r["n_applied"] == 2 and r["status"][-1] == 7
