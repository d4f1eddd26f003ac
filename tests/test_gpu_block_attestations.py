"""process_attestation for a run of blocks on the GPU (b2_block_attestations / _dev, Engine.block_attestations / _dev,
Spec.process_block_attestations) against tests/block_attestations_oracle.py: every status 1-11, the flag boundaries, both ABI forms,
order-exact credit across blocks, block-atomic failure, epoch 0, committee counts that differ between the two epochs, the RLC verify mode,
the device guards, the host form's refusals and a 2 048-member committee at bits_stride 256.  Signatures are made on the GPU by b2_sign
with each aggregate's summed secret key; their verdicts are known by construction (the right key sum over the right message, or a planted
corruption).  The 8 process_attestation cases of tests/golden/literal_spec.json are replayed as one-attestation blocks."""
import hashlib

import numpy as np
import pytest
import torch

import block_attestations_oracle as O
import test_golden as TG
from oracle.bls12_381 import R
from pos_evolution_b200._lib import B2_EINVAL, B2Error
from pos_evolution_b200.engine import Engine

pytestmark = pytest.mark.gpu

INC, PER_INC = 10**9, 977
DOMAINS = bytes([1] * 32) + bytes([2] * 32)


def _h(b):
    return hashlib.sha256(b).digest()


class World:
    """n_val validators (secret key i + 1), the committees of epochs e - 1 and e (sizes drawn from `sizes`), a chain of 2 * spe roots"""

    def __init__(self, eng, n_val, spe, e, cps_prev, cps_cur, sizes, stride, seed):
        rng = np.random.default_rng(seed)
        self.eng, self.n_val, self.spe, self.e, self.cps_prev, self.cps_cur, self.stride = eng, n_val, spe, e, cps_prev, cps_cur, stride
        self.sks = [i + 1 for i in range(n_val)]
        self.eff = (rng.choice([32, 32, 31, 24, 16], size=n_val) * 10**9).astype(np.uint64)
        eng.registry_load(eng.sk_to_pk(self.sks), self.eff)
        members, off = [], [0]
        for E, cps in ((e - 1, cps_prev), (e, cps_cur)):
            if cps == 0:
                continue
            perm = rng.permutation(n_val)
            k = 0
            for _ in range(cps * spe):
                size = int(rng.choice(sizes))
                members += perm[k:k + size].tolist()
                k += size
                off.append(len(members))
        self.members, self.off = np.array(members, np.uint32), np.array(off, np.uint32)
        self.roots = [_h(b"root" + bytes([seed, s])) for s in range(2 * spe)]
        self.justified = ((max(e, 2) - 2).to_bytes(8, "little") + _h(b"j-prev") + (max(e, 1) - 1).to_bytes(8, "little") + _h(b"j-cur"))
        self.good = {}

    def root(self, slot):
        return self.roots[slot + self.spe - self.e * self.spe]

    def committee(self, slot, index):
        E = slot // self.spe
        cps = self.cps_cur if E == self.e else self.cps_prev
        c = (self.cps_prev * self.spe if E == self.e else 0) + (slot - E * self.spe) * cps + index
        return self.members[self.off[c]:self.off[c + 1]].tolist()

    def att(self, slot, index, bits=None, head=None, target=None, source=None, tepoch=None, corrupt=False, size=None):
        """the encoding of a signed attestation of committee (slot, index), right unless told otherwise"""
        E = slot // self.spe
        tepoch = E if tepoch is None else tepoch
        com = self.committee(slot, index) if index < (self.cps_cur if E == self.e else self.cps_prev) else [0] * (size or 4)
        bits = [True] * len(com) if bits is None else list(bits)
        if source is None:
            source = self.justified[40:80] if tepoch == self.e else self.justified[0:40]
        d = O.data128(slot, index, self.root(slot) if head is None else head, int.from_bytes(source[:8], "little"), source[8:], tepoch,
                      self.root(tepoch * self.spe) if 0 <= tepoch * self.spe - (self.e - 1) * self.spe < 2 * self.spe and target is None
                      else (target or bytes(32)))
        sel = sorted(set(v for v, b in zip(com, bits) if b))
        msg = O.signing_root(d, DOMAINS[32:] if tepoch == self.e else DOMAINS[:32])
        sk = (sum(self.sks[v] for v in sel) + (1 if corrupt else 0)) % R or 1
        sig = bytes(self.eng.sign([sk], [0], np.frombuffer(msg, np.uint8).reshape(1, 32))[0])
        if not corrupt:
            self.good[(tuple(sel), msg)] = sig
        return O.encode(bits, d, sig)

    def verify(self, idx, root, sig):
        return self.good.get((tuple(idx), root)) == bytes(sig)

    def tables(self, seed):
        rng = np.random.default_rng(seed)
        return [(rng.integers(0, 8, self.n_val) * (rng.random(self.n_val) < 0.3)).astype(np.uint8) for _ in range(2)]

    def args(self, blocks, slots):
        wire, woff, block_off = O.layout(blocks)
        return dict(wire=wire, woff=woff, block_off=block_off, block_slot=np.array(slots, np.uint64), members=self.members, off=self.off,
                    cps_prev=self.cps_prev, cps_cur=self.cps_cur, chain_roots=np.frombuffer(b"".join(self.roots), np.uint8),
                    justified80=self.justified, domains64=DOMAINS, slots_per_epoch=self.spe, min_inclusion_delay=1, bits_stride=self.stride,
                    increment=INC, base_reward_per_increment=PER_INC)

    def host(self, a, t):
        self.eng.participation_load(0, t[0])
        self.eng.participation_load(1, t[1])
        r = self.eng.block_attestations(**a)
        return r, self.eng.participation_read(0), self.eng.participation_read(1)

    def dev(self, a, t):
        eng = self.eng
        eng.participation_load(0, t[0])
        eng.participation_load(1, t[1])
        n, nb = len(a["woff"]) - 1, len(a["block_off"]) - 1
        T = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dtype=dt).copy()).cuda()      # noqa: E731
        w = T(np.frombuffer(a["wire"], np.uint8), np.uint8)
        outs = [torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda"),
                torch.zeros(n, dtype=torch.uint64, device="cuda"), torch.zeros(nb, dtype=torch.int32, device="cuda"),
                torch.zeros(nb, dtype=torch.uint32, device="cuda"), torch.zeros(nb, dtype=torch.uint64, device="cuda"),
                torch.zeros(1, dtype=torch.uint32, device="cuda")]
        eng.block_attestations_dev(w, T(a["woff"], np.uint32), T(a["block_off"], np.uint32), T(a["block_slot"], np.uint64),
                                   T(a["members"], np.uint32), T(a["off"], np.uint32), a["cps_prev"], a["cps_cur"], T(a["chain_roots"], np.uint8),
                                   a["justified80"], a["domains64"], a["slots_per_epoch"], a["min_inclusion_delay"], a["bits_stride"], INC, PER_INC,
                                   *outs)
        torch.cuda.synchronize()
        o = [x.cpu().numpy() for x in outs]
        return (o[0], o[1], o[2], o[3], o[4], o[5], int(o[6][0])), eng.participation_read(0), eng.participation_read(1)

    def oracle(self, a, t):
        return O.run(a["wire"], a["woff"], a["block_off"], a["block_slot"], self.members, self.off, self.cps_prev, self.cps_cur, self.roots,
                     self.justified, DOMAINS, self.spe, 1, self.stride, self.eff, INC, PER_INC, t[0].tolist(), t[1].tolist(), self.verify)


def same(got, o):
    (st, mask, num, bst, bfirst, brew, napp), t0, t1 = got
    assert np.asarray(st).tolist() == o["status"].tolist()
    assert np.asarray(mask).tolist() == o["flag_mask"].tolist()
    assert np.asarray(num).tolist() == o["numerator"].tolist()
    assert np.asarray(bst).tolist() == o["block_status"].tolist()
    assert np.asarray(bfirst).tolist() == o["block_first"].tolist()
    assert np.asarray(brew).tolist() == o["block_reward"].tolist()
    assert int(napp) == o["n_applied"]
    assert t0.tolist() == o["part_cur"] and t1.tolist() == o["part_prev"]


def both_forms(W, blocks, slots, seed=0):
    a, t = W.args(blocks, slots), W.tables(seed)
    o = W.oracle(a, t)
    same(W.host(a, t), o)
    same(W.dev(a, t), o)
    return o


@pytest.fixture(scope="module")
def W():
    # e = 3 on 4-slot epochs (slots 12-15; e - 1 = slots 8-11), 2 committees per slot before, 3 in e; ragged committees of 3-24
    return World(Engine(0), 400, 4, 3, 2, 3, list(range(3, 25)), 4, 1)


def _valid_block(W, s):
    return [W.att(s - 1, 0), W.att(s - 1, 1, bits=[j % 2 == 0 for j in range(len(W.committee(s - 1, 1)))]), W.att(s - 3, 1), W.att(s - 4, 0)]


def test_every_status_through_both_forms(W):
    s = 14
    bad = [W.att(13, 0)[:200], W.att(13, 0)[:228], W.att(13, 2, bits=[True] * 33), W.att(5, 0, tepoch=1), W.att(9, 0, tepoch=3),
           W.att(9, 1), W.att(13, 3), W.att(13, 0, bits=[True] * (len(W.committee(13, 0)) - 1)), W.att(13, 0, source=W.justified[:40]),
           W.att(13, 1, bits=[False] * len(W.committee(13, 1))), W.att(12, 2, corrupt=True)]
    o = both_forms(W, [_valid_block(W, 13), [W.att(13, 1)] + bad, _valid_block(W, 15)], [13, s, 15])
    assert o["status"].tolist()[4:16] == [0] + list(range(1, 12)) and o["n_applied"] == 1 and o["block_status"].tolist() == [0, 1, 2]
    assert o["block_first"].tolist() == [0xFFFFFFFF, 1, 0xFFFFFFFF]


def test_flag_boundaries(W):
    """delays 1, 2 = isqrt(4), 3, 4 = SLOTS_PER_EPOCH into the current and the previous table, head and target mismatches; delay 5 fails"""
    blk = [W.att(15 - d, k % 2) for k, d in enumerate((1, 2, 3, 4))]
    blk += [W.att(14, 2, head=_h(b"h")), W.att(14, 1, target=_h(b"t"), head=_h(b"h"))]
    o = both_forms(W, [blk], [15])
    assert o["flag_mask"].tolist() == [7, 3, 2, 2, 3, 1] and o["n_applied"] == 1
    o = both_forms(W, [blk + [W.att(10, 0)]], [15])
    assert o["status"].tolist()[-1] == 6 and o["n_applied"] == 0


def test_order_exact_credit_across_blocks(W):
    """overlapping aggregates of one committee over three blocks: each later one earns only the flags still unset"""
    com = len(W.committee(12, 0))
    half = [j < com // 2 for j in range(com)]
    blocks = [[W.att(12, 0, bits=half), W.att(12, 0, bits=[not b for b in half]), W.att(11, 0)], [W.att(12, 0), W.att(12, 0)],
              [W.att(12, 0, bits=half), W.att(13, 1), W.att(11, 0)]]
    o = both_forms(W, blocks, [13, 14, 15], seed=5)
    assert o["n_applied"] == 3 and o["status"].tolist() == [0] * 8
    assert o["numerator"].tolist()[3:6] == [0, 0, 0] and o["numerator"][7] == 0 and o["numerator"][0] > 0


def test_block_atomic_failure(W):
    """an invalid block in the middle: the tables hold exactly the blocks before it, its rewards and the later blocks' are 0"""
    blocks = [_valid_block(W, 13), [W.att(13, 2), W.att(13, 1, corrupt=True), W.att(13, 0)], _valid_block(W, 15)]
    o = both_forms(W, blocks, [13, 14, 15], seed=9)
    assert o["n_applied"] == 1 and o["block_reward"].tolist()[1:] == [0, 0] and o["numerator"].tolist()[4:] == [0] * 7
    a, t = W.args(blocks[:1], [13]), W.tables(9)
    first = W.host(a, t)
    bad = W.host(W.args(blocks, [13, 14, 15]), t)
    assert first[1].tolist() == bad[1].tolist() and first[2].tolist() == bad[2].tolist()


def test_rlc_mode_gives_identical_outputs(W):
    blocks = [_valid_block(W, 13), [W.att(13, 2), W.att(12, 1, corrupt=True)] + _valid_block(W, 14), _valid_block(W, 15)]
    a, t = W.args(blocks, [13, 14, 15]), W.tables(3)
    ref = W.host(a, t)
    W.eng.set_verify_mode(True, bytes(range(32)))
    try:
        got = W.host(a, t)
    finally:
        W.eng.set_verify_mode(False)
    for x, y in zip(ref[0], got[0]):
        assert np.asarray(x).tolist() == np.asarray(y).tolist()
    assert ref[1].tolist() == got[1].tolist() and ref[2].tolist() == got[2].tolist()
    same(got, W.oracle(a, t))


def test_epoch_zero():
    eng = Engine(0)
    W0 = World(eng, 120, 4, 0, 0, 3, list(range(4, 10)), 2, 2)
    blocks = [[W0.att(0, 0), W0.att(0, 2)], [W0.att(1, 1), W0.att(0, 0)], [W0.att(2, 2), W0.att(1, 0, tepoch=1)]]
    o = both_forms(W0, blocks, [1, 2, 3])
    assert o["status"].tolist() == [0, 0, 0, 0, 0, 4] and o["n_applied"] == 2 and o["block_status"].tolist() == [0, 0, 1]
    o = both_forms(W0, blocks[:2] + [blocks[2][:1]], [1, 2, 3])
    assert o["n_applied"] == 3


def test_two_thousand_member_committee_at_stride_256():
    eng = Engine(0)
    W2 = World(eng, 8192, 4, 5, 1, 1, [2048], 256, 4)         # epoch 5 = slots 20-23; four committees of 2 048 per epoch
    some = W2.att(20, 0, bits=[j % 3 == 0 for j in range(2048)])
    o = both_forms(W2, [[some, W2.att(17, 0, bits=[j >= 1024 for j in range(2048)])], [W2.att(21, 0), W2.att(19, 0, bits=[True] * 2047)]],
                   [21, 22])
    assert o["status"].tolist() == [0, 0, 0, 8] and o["n_applied"] == 1 and o["flag_mask"].tolist()[:3] == [7, 2, 7]


def _dev_call(W, a, t, mutate):
    a = dict(a)
    mutate(a)
    W.eng.guard_flags()
    got = W.dev(a, t)
    return got, W.eng.guard_flags()


def test_device_guards(W):
    blocks = [_valid_block(W, 13), _valid_block(W, 14)]
    a, t = W.args(blocks, [13, 14]), W.tables(2)
    # a reversed woff row: status 1, the block is invalid
    def woff(x):
        x["woff"] = x["woff"].copy()
        x["woff"][5] = x["woff"][6] + 1
    got, g = _dev_call(W, a, t, woff)
    assert got[0][0][5] == 1 and got[0][3].tolist() == [0, 1] and got[0][6] == 1 and g & 2
    # the row of committee (12, 0) ends past the members: status 8
    def off(x):
        x["off"] = x["off"].copy()
        x["off"][W.cps_prev * W.spe + 1] = len(x["members"]) + 5
    got, g = _dev_call(W, a, t, off)
    assert got[0][0][0] == 8 and got[0][6] == 0 and g & 2
    # a reversed block row: that block is invalid, nothing of it applied
    def boff(x):
        x["block_off"] = x["block_off"].copy()
        x["block_off"][1] = 9
    got, g = _dev_call(W, a, t, boff)
    assert got[0][3].tolist() == [1, 1] and got[0][6] == 0 and g & 2
    assert got[1].tolist() == t[0].tolist() and got[2].tolist() == t[1].tolist()
    # block slots that do not increase: the second block is invalid
    def slots(x):
        x["block_slot"] = np.array([13, 13], np.uint64)
    got, g = _dev_call(W, a, t, slots)
    assert got[0][3].tolist() == [0, 1] and got[0][6] == 1 and g & 2
    # a member index past the registry: FastAggregateVerify fails (11)
    def member(x):
        x["members"] = x["members"].copy()
        x["members"][x["off"][W.cps_prev * W.spe]] = W.n_val + 7        # the first member of committee (12, 0)
    blk = [[W.att(12, 0)]]
    a2 = W.args(blk, [13])
    got, g = _dev_call(W, a2, t, member)
    assert got[0][0].tolist() == [11] and got[0][6] == 0 and g & 1


def test_host_refusals_change_nothing(W):
    blocks = [_valid_block(W, 13), _valid_block(W, 14)]
    a, t = W.args(blocks, [13, 14]), W.tables(4)
    W.eng.participation_load(0, t[0])
    W.eng.participation_load(1, t[1])
    bad = []
    for key, value in (("woff", None), ("block_off", None), ("off", None), ("block_slot", np.array([14, 13], np.uint64)),
                       ("block_slot", np.array([15, 16], np.uint64)), ("cps_prev", 3), ("bits_stride", 0), ("bits_stride", 257),
                       ("bits_stride", 2)):
        x = dict(a)
        if value is None:
            x[key] = x[key].copy()
            x[key][1], x[key][2] = x[key][2], x[key][1]      # decreasing
        else:
            x[key] = value
        bad.append(x)
    x = dict(a)
    x["woff"] = x["woff"].copy()
    x["woff"][-1] = len(x["wire"]) + 1
    bad.append(x)
    x = dict(a)
    x["block_off"] = x["block_off"][:2].copy()                 # ends before n_att
    x["block_slot"] = x["block_slot"][:1]
    bad.append(x)
    for x in bad:
        with pytest.raises(B2Error) as err:
            W.eng.block_attestations(**x)
        assert err.value.code == B2_EINVAL
    assert W.eng.participation_read(0).tolist() == t[0].tolist() and W.eng.participation_read(1).tolist() == t[1].tolist()
    # e = 0 with committees of a previous epoch, and no blocks
    x = dict(a, block_slot=np.array([1, 2], np.uint64))
    with pytest.raises(B2Error):
        W.eng.block_attestations(**x)
    with pytest.raises(B2Error):
        W.eng.block_attestations(**dict(a, block_off=np.zeros(1, np.uint32), block_slot=np.zeros(0, np.uint64)))
    with pytest.raises(B2Error):
        W.eng.block_attestations(**dict(a, wire=b"", woff=np.zeros(1, np.uint32), block_off=np.zeros(2, np.uint32), block_slot=[13]))
    assert W.eng.participation_read(0).tolist() == t[0].tolist() and W.eng.participation_read(1).tolist() == t[1].tolist()
    # no registry; a registry without participation tables
    eng = Engine(0)
    for _ in range(2):
        with pytest.raises(B2Error) as err:
            eng.block_attestations(**a)
        assert err.value.code == B2_EINVAL
        eng.registry_load(eng.sk_to_pk([1, 2, 3]), np.full(3, 32 * 10**9, np.uint64))


def test_golden_process_attestation_cases_as_blocks():
    from pos_evolution_b200 import spec as PS
    pspec = PS.Spec(PS.MINIMAL, engine=Engine(0))
    _, ostate = TG._state(TG.PKS)
    for case in TG.G["process_attestation"]:
        st = TG._pstate(PS, ostate)
        proposer = pspec.get_beacon_proposer_index(st)
        n, statuses = pspec.process_block_attestations(st, [PS.BlockAttestations(st.slot, proposer, _h(b"block"), [TG._att(PS, case["attestation"])])])
        if case["result"] == "ok":
            assert n == 1 and statuses[0].tolist() == [0]
            assert st.balances == case["balances"]
            assert st.current_epoch_participation == case["current_epoch_participation"]
            assert st.previous_epoch_participation == case["previous_epoch_participation"]
        else:
            assert n == 0 and statuses[0][0] != 0, case["name"]
            assert st.balances == ostate.balances and st.current_epoch_participation == ostate.current_epoch_participation


class KnownBLS:
    """FastAggregateVerify for oracle.spec: true for the signatures made right (by the secret keys of exactly these members, over this
    message), which the test records as it makes them"""
    good = {}

    @staticmethod
    def FastAggregateVerify(pubkeys, msg, sig):
        return KnownBLS.good.get((tuple(bytes(p) for p in pubkeys), bytes(msg))) == bytes(sig)


def test_spec_multi_block_runs_match_the_spec_block_by_block():
    """Spec.process_block_attestations over four blocks of one epoch whose later attestations vote for earlier blocks of the run (the
    chain roots come from blocks[k].root), each block with its own proposer, against oracle.spec.process_attestation block by block:
    every block valid, then a run whose third block holds a bad signature"""
    import copy

    import scenarios
    from oracle import spec as OS
    from pos_evolution_b200 import spec as PS
    eng = Engine(0)
    pspec = PS.Spec(PS.MINIMAL, engine=eng)
    ospec = OS.Spec(OS.MINIMAL, bls_module=KnownBLS)
    spe, H = OS.MINIMAL.SLOTS_PER_EPOCH, OS.MINIMAL.SLOTS_PER_HISTORICAL_ROOT
    _, base = scenarios.minimal_state(64, slot=17, pks=TG.PKS)
    base.previous_justified_checkpoint = OS.Checkpoint(0, _h(b"j0"))
    base.current_justified_checkpoint = OS.Checkpoint(1, _h(b"j1"))
    slots = [17, 19, 20, 22]
    roots = [_h(b"run" + bytes([s])) for s in slots]

    def root(s):
        return bytes(base.block_roots[s % H]) if s < slots[0] else [r for r, b in zip(roots, slots) if b <= s][-1]

    def att(s, index, bits=None, corrupt=False):
        E = s // spe
        com = ospec.get_beacon_committee(base, s, index)
        bits = [True] * len(com) if bits is None else bits
        src = base.current_justified_checkpoint if E == 2 else base.previous_justified_checkpoint
        data = OS.AttestationData(s, index, root(s), src, OS.Checkpoint(E, root(E * spe)))
        msg = ospec.compute_signing_root(data, ospec.get_domain(base, OS.DOMAIN_BEACON_ATTESTER, E))
        sel = sorted(set(v for v, b in zip(com, bits) if b))
        sk = (sum(scenarios.secret_key(v) for v in sel) + (1 if corrupt else 0)) % R
        sig = bytes(eng.sign([sk], [0], np.frombuffer(msg, np.uint8).reshape(1, 32))[0])
        if not corrupt:
            KnownBLS.good[(tuple(bytes(TG.PKS[v]) for v in sel), msg)] = sig
        return OS.Attestation(bits, data, sig)

    def product(a):
        d = a.data
        return PS.Attestation(list(a.aggregation_bits), PS.AttestationData(d.slot, d.index, d.beacon_block_root, PS.Checkpoint(d.source.epoch, d.source.root),
                                                                           PS.Checkpoint(d.target.epoch, d.target.root)), a.signature)

    def check(blocks):
        st, failed = copy.deepcopy(base), None
        for k, s in enumerate(slots):
            if k:
                for t in range(slots[k - 1], s):
                    st.block_roots[t % H] = roots[k - 1]
            st.slot = s
            before = copy.deepcopy(st)
            try:
                for a in blocks[k]:
                    ospec.process_attestation(st, a)
            except AssertionError:
                st, failed = before, k
                break
        proposers = []
        for s in slots:
            at = copy.copy(base)
            at.slot = s
            proposers.append(ospec.get_beacon_proposer_index(at))
        assert len(set(proposers)) > 1
        ps = TG._pstate(PS, base)
        n, statuses = pspec.process_block_attestations(ps, [PS.BlockAttestations(s, p, r, [product(a) for a in blk])
                                                            for s, p, r, blk in zip(slots, proposers, roots, blocks)])
        assert n == (len(slots) if failed is None else failed)
        assert ps.balances == st.balances
        assert ps.current_epoch_participation == st.current_epoch_participation
        assert ps.previous_epoch_participation == st.previous_epoch_participation
        assert ps.slot == base.slot and ps.block_roots == base.block_roots
        return n, statuses

    run = [[att(16, 0), att(16, 1), att(13, 0)],
           [att(18, 0), att(17, 1), att(15, 1)],                      # heads at slots 17 and 18: the run's first block
           [att(19, 0), att(18, 1, bits=[True, False, True, False]), att(18, 0)],
           [att(21, 1), att(20, 0), att(19, 1)]]
    n, statuses = check(run)
    assert n == 4 and all(not s.any() for s in statuses)
    run[2] = [att(19, 0), att(18, 1, corrupt=True), att(18, 0)]
    n, statuses = check(run)
    assert n == 2 and statuses[2].tolist() == [0, 11, 0]
