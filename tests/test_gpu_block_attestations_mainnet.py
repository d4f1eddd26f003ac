"""process_attestation for a run of blocks on the GPU (b2_block_attestations / _dev) at mainnet shape, against
tests/block_attestations_oracle.py byte for byte through both ABI forms and both participation tables:

  (a) a full 32-slot epoch of 32 blocks x 128 aggregates with 64 committees per slot over 2^17 validators: both tables, delays 1-32,
      re-inclusions, disjoint halves, supersets, head and target mismatches, the first and last committees of both epochs; again in the
      RLC verify mode.  The test checks that it reaches what it claims (more than 1 024 attestations, every mask the rules allow, a flag
      won past attestation 1 024, a re-inclusion that earns nothing);
  (b) block-atomic failure on that epoch: a bad signature at the last attestation, a bad block 0, two bad blocks;
  (c) the 5-slot source and 32-slot target windows, delay 33 and the first slot of the previous epoch;
  (d) empty blocks first, in the middle, last, in a row, before an invalid block;
  (e) each attestation's numerator floored on its own (:752-754), with effective balances that vary by validator and some below
      EFFECTIVE_BALANCE_INCREMENT;
  (f) committee sizes 1-2 048 at a tight bits_stride and at 256, with first-bit, last-bit, full and alternating bit rows;
  (g) the full 2^20-validator epoch on the mainnet preset through Spec.block_attestations_inputs;
and Spec.process_block_attestations on the mainnet preset against oracle.spec.process_attestation block by block and against
Spec.process_attestations, over a run with skipped slots, a repeated proposer, an empty block, a fork at the run's epoch and a mid-run
invalid block.  Signatures are made on the GPU by b2_sign with each aggregate's summed secret key, a whole call's aggregates in one batch.
Run on an H100:
    python -m pytest tests/test_gpu_block_attestations_mainnet.py -m gpu"""
import copy
import hashlib

import numpy as np
import pytest

import block_attestations_oracle as O
import scenarios
import test_golden as TG
from oracle.bls12_381 import R
from pos_evolution_b200.engine import Engine
from test_gpu_block_attestations import DOMAINS, INC, KnownBLS, World, both_forms, same

pytestmark = pytest.mark.gpu

SPE = 32
E = 3
START = E * SPE                                    # slots 96-127; e - 1 = slots 64-95
NONE = 0xFFFFFFFF
OTHER_HEAD, OTHER_TARGET = hashlib.sha256(b"other head").digest(), hashlib.sha256(b"other target").digest()


class Batch:
    """Attestations of one World, signed together: add() returns a handle, sign() makes every signature in one Engine.sign call and
    returns the encodings by handle.  The right signatures are recorded in World.good, as World.att does."""

    def __init__(self, W):
        self.W, self.items = W, []

    def add(self, slot, index, bits=None, head=None, target=None, corrupt=False):
        W = self.W
        tepoch = slot // W.spe
        com = W.committee(slot, index)
        bits = [True] * len(com) if bits is None else list(bits)
        source = W.justified[40:80] if tepoch == W.e else W.justified[0:40]
        d = O.data128(slot, index, W.root(slot) if head is None else head, int.from_bytes(source[:8], "little"), source[8:], tepoch,
                      W.root(tepoch * W.spe) if target is None else target)
        sel = sorted(set(v for v, b in zip(com, bits) if b))
        msg = O.signing_root(d, DOMAINS[32:] if tepoch == W.e else DOMAINS[:32])
        self.items.append((bits, d, sel, msg, (sum(W.sks[v] for v in sel) + (1 if corrupt else 0)) % R or 1, corrupt))
        return len(self.items) - 1

    def sign(self):
        sigs = self.W.eng.sign([it[4] for it in self.items], np.arange(len(self.items), dtype=np.uint32),
                               np.frombuffer(b"".join(it[3] for it in self.items), np.uint8).reshape(-1, 32))
        wires = []
        for (bits, d, sel, msg, _, corrupt), sig in zip(self.items, sigs):
            if not corrupt:
                self.W.good[(tuple(sel), msg)] = bytes(sig)
            wires.append(O.encode(bits, d, bytes(sig)))
        return wires


# ------------------------------------------------------------------------------------------------ (a), (b): a full mainnet-shaped epoch
@pytest.fixture(scope="module")
def epoch():
    """32 blocks at START .. START + 31, 128 attestations each.  Per block at slot s:
      - every committee of slot s - 1 (delay 1): in full, except a head mismatch (i % 16 == 5), a target mismatch (i % 16 == 9), the first
        half (i % 8 == 3) and the first quarter (i % 16 == 13);
      - the other halves of slot s - 3 (i in 3, 19, 35, 51: delay 3) and of slot s - 7 (i in 11, 27, 43, 59: delay 7);
      - supersets of the quarters: the first half of slot s - 2 and the whole of slot s - 6 (i in 13, 29, 45, 61);
      - eight exact re-inclusions of aggregates of the eight blocks before;
      - four target mismatches at delays 6-32, four at delays 2-5, four head mismatches at delays 2-32;
      - committees drawn at delays 2-32 with about 70 % of their bits, up to 128;
    each block's list shuffled.  Block 0 also carries (start(e - 1), 0), the first committee of the previous epoch, at delay 32."""
    eng = Engine(0)
    W = World(eng, 1 << 17, SPE, E, 64, 64, list(range(40, 65)), 8, 7)
    rng = np.random.default_rng(21)
    B = Batch(W)
    plan, key, delay = [], {}, {}

    def add(k, slot, i, **kw):
        h = B.add(slot, i, **kw)
        key[h], delay[h] = (slot, i), START + k - slot
        plan[k].append(h)
        return h

    reinc = []
    for k in range(SPE):
        s = START + k
        plan.append([])
        for i in range(64):
            n = len(W.committee(s - 1, i))
            if i % 16 == 5:
                add(k, s - 1, i, head=OTHER_HEAD)
            elif i % 16 == 9:
                add(k, s - 1, i, target=OTHER_TARGET)
            elif i % 8 == 3:
                add(k, s - 1, i, bits=[j < n // 2 for j in range(n)])
            elif i % 16 == 13:
                add(k, s - 1, i, bits=[j < n // 4 for j in range(n)])
            else:
                add(k, s - 1, i)
        for d, idx in ((3, (3, 19, 35, 51)), (7, (11, 27, 43, 59))):
            for i in idx:
                n = len(W.committee(s - d, i))
                add(k, s - d, i, bits=[j >= n // 2 for j in range(n)])
        for i in (13, 29, 45, 61):
            n = len(W.committee(s - 2, i))
            add(k, s - 2, i, bits=[j < n // 2 for j in range(n)])
            add(k, s - 6, i)
        if k:
            earlier = [h for b in plan[max(0, k - 8):k] for h in b if key[h][0] >= s - SPE]
            for h in rng.choice(earlier, 8, replace=False):
                plan[k].append(int(h))
                reinc.append((k, int(h)))
        for lo, hi, kw in ((6, 32, dict(target=OTHER_TARGET)), (2, 5, dict(target=OTHER_TARGET)), (2, 32, dict(head=OTHER_HEAD))):
            for _ in range(4):
                add(k, s - int(rng.integers(lo, hi + 1)), int(rng.integers(0, 64)), **kw)
        if k == 0:
            add(k, START - SPE, 0)
        while len(plan[k]) < 128:
            slot, i = s - int(rng.integers(2, SPE + 1)), int(rng.integers(0, 64))
            bits = rng.random(len(W.committee(slot, i))) < 0.7
            bits[int(rng.integers(0, len(bits)))] = True
            add(k, slot, i, bits=bits.tolist())
        plan[k] = [plan[k][j] for j in rng.permutation(len(plan[k]))]
    # the planted failures of (b): a wrong key sum each
    bad = {name: B.add(slot, i, corrupt=True) for name, slot, i in (("last", START + 30, 1), ("first", START - 1, 2),
                                                                     ("b10", START + 9, 0), ("b20", START + 19, 0))}
    wires = B.sign()
    blocks = [[wires[h] for h in p] for p in plan]
    slots = [START + k for k in range(SPE)]
    yield dict(W=W, blocks=blocks, slots=slots, plan=plan, key=key, delay=delay, reinc=reinc, bad={k: wires[h] for k, h in bad.items()})
    eng.close()


def test_full_mainnet_epoch(epoch):
    W, blocks, slots, plan, key = epoch["W"], epoch["blocks"], epoch["slots"], epoch["plan"], epoch["key"]
    o = both_forms(W, blocks, slots, seed=31)
    n = sum(len(b) for b in blocks)
    flat = [h for p in plan for h in p]
    assert n == 4096 > 1024 and all(len(b) > 32 for b in blocks)
    assert o["n_applied"] == SPE and not o["status"].any() and not o["block_status"].any()
    assert o["block_first"].tolist() == [NONE] * SPE and (o["block_reward"] > 0).all()
    # what the epoch reaches: every inclusion delay, both tables, every mask the rules allow
    assert sorted(set(epoch["delay"][h] for h in flat)) == list(range(1, SPE + 1))
    assert {key[h][0] >= START for h in flat} == {True, False}
    assert set(o["flag_mask"].tolist()) == {0, 1, 2, 3, 7}
    extremes = {(START - SPE, 0), (START - 1, 63), (START, 0), (START + 30, 63)}
    assert extremes <= {key[h] for h in flat}
    # a flag election won past attestation 1 024 against an earlier aggregate of the same committee, and re-inclusions that earn nothing
    first_seen = {}
    for a, h in enumerate(flat):
        first_seen.setdefault(key[h], a)
    assert any(a > 1024 and o["numerator"][a] > 0 and first_seen[key[h]] < a for a, h in enumerate(flat))
    offs = np.concatenate([[0], np.cumsum([len(p) for p in plan])])
    reinc_pos = [int(offs[k]) + plan[k].index(h) for k, h in epoch["reinc"]]
    assert len(reinc_pos) >= 8 * 31 and all(o["numerator"][a] == 0 for a in reinc_pos)
    # the RLC verify mode: the same outputs
    a, t = W.args(blocks, slots), W.tables(31)
    W.eng.set_verify_mode(True, bytes(range(32)))
    try:
        got = W.host(a, t)
    finally:
        W.eng.set_verify_mode(False)
    same(got, o)


@pytest.mark.parametrize("case", ["last", "first", "two"])
def test_block_atomic_failure_at_scale(epoch, case):
    """a bad signature at attestation 4 095 (the last of block 31), one in block 0, or one in each of blocks 10 and 20: the tables hold
    exactly the blocks before the first invalid one, run alone"""
    W, slots = epoch["W"], epoch["slots"]
    blocks = [list(b) for b in epoch["blocks"]]
    bad = epoch["bad"]
    if case == "last":
        blocks[31][-1] = bad["last"]
        want = 31
    elif case == "first":
        blocks[0][5] = bad["first"]
        want = 0
    else:
        blocks[10][7], blocks[20][100] = bad["b10"], bad["b20"]
        want = 10
    o = both_forms(W, blocks, slots, seed=33)
    assert o["n_applied"] == want and o["block_status"][want] == 1 and o["status"].tolist().count(11) == (2 if case == "two" else 1)
    assert o["block_status"].tolist()[want + 1:] == [1 if (case == "two" and b == 20) else 2 for b in range(want + 1, SPE)]
    assert o["block_reward"][want:].tolist() == [0] * (SPE - want)
    t = W.tables(33)
    got = W.host(W.args(blocks, slots), t)
    if want:
        prefix = W.host(W.args(blocks[:want], slots[:want]), t)
        assert prefix[1].tolist() == got[1].tolist() and prefix[2].tolist() == got[2].tolist()
    else:
        assert got[1].tolist() == t[0].tolist() and got[2].tolist() == t[1].tolist()


# ------------------------------------------------------------------------------------------------ (c), (d), (e): 32-slot epochs, 4 committees a slot
@pytest.fixture(scope="module")
def M():
    """4 096 validators, 4 committees of 8-24 per slot of epochs 2 and 3, bits_stride 3.  Effective balances vary: 1-32 increments, and a
    few validators (every member of committee (START + 3, 0) among them) hold less than one increment"""
    eng = Engine(0)
    W = World(eng, 4096, SPE, E, 4, 4, list(range(8, 25)), 3, 9)
    rng = np.random.default_rng(41)
    W.eff = (rng.integers(1, 33, W.n_val) * INC).astype(np.uint64)
    low = np.array(sorted(set(W.committee(START + 3, 0)) | set(rng.choice(W.n_val, 100, replace=False).tolist())))
    W.eff[low] = rng.integers(1, INC, len(low)).astype(np.uint64)
    W.low = set(low.tolist())
    eng.registry_update_balances(W.eff, np.ones(W.n_val, np.uint8))
    yield W
    eng.close()


def test_inclusion_windows_at_32_slots(M):
    """block start(e): the previous table at delays 1, 2, 5, 6, 31, 32, a head mismatch at delay 1, target mismatches at delays 5 and 6;
    block start(e) + 31: the current table at delays 1, 2, 5, 6, 31 and the same mismatches.  A target-e attestation at delay 32 is
    included in epoch e + 1, where e is the previous epoch: the previous table's delay 32 covers it."""
    last = START + SPE - 1
    blocks = [[M.att(START - d, d % 4) for d in (1, 2, 5, 6, 31, 32)], [M.att(last - d, d % 4) for d in (1, 2, 5, 6, 31)]]
    for k, s in enumerate((START, last)):
        blocks[k] += [M.att(s - 1, 1, head=OTHER_HEAD), M.att(s - 5, 2, target=OTHER_TARGET), M.att(s - 6, 2, target=OTHER_TARGET)]
    o = both_forms(M, blocks, [START, last], seed=3)
    assert o["n_applied"] == 2 and not o["status"].any()
    assert o["flag_mask"].tolist() == [7, 3, 3, 2, 2, 2, 3, 1, 0] + [7, 3, 3, 2, 2, 3, 1, 0]
    assert o["numerator"][8] == 0 and o["numerator"][16] == 0
    # a mask-0 attestation alone: valid, no flag set, nothing earned
    for s, w in ((START, blocks[0][8]), (last, blocks[1][7])):
        a, t = M.args([[w]], [s]), M.tables(4)
        o = both_forms(M, [[w]], [s], seed=4)
        got = M.host(a, t)
        assert o["status"].tolist() == [0] and o["flag_mask"].tolist() == [0] and o["numerator"].tolist() == [0]
        assert got[1].tolist() == t[0].tolist() and got[2].tolist() == t[1].tolist()
    # start(e - 1) at start(e) (delay 32) is valid; one slot later (delay 33) it is status 6
    w = M.att(START - SPE, 0)
    o = both_forms(M, [[w]], [START])
    assert o["status"].tolist() == [0] and o["flag_mask"].tolist() == [2]
    o = both_forms(M, [[M.att(START - 1, 0)], [w]], [START, START + 1])
    assert o["n_applied"] == 1 and o["status"].tolist() == [0, 6] and o["block_status"].tolist() == [0, 1]
    o = both_forms(M, [[M.att(START - SPE + 1, 3)]], [START + 2])
    assert o["status"].tolist() == [6] and o["n_applied"] == 0


@pytest.mark.parametrize("shape", ["first_middle_last", "in_a_row", "only_the_last", "invalid_after_empty", "empty_after_invalid"])
def test_empty_blocks(M, shape):
    """empty blocks: status 0 when applied (2 after an invalid block), block_first 0xFFFFFFFF, reward 0, no guard bit"""
    a1, a2, a3, a4 = M.att(START + 3, 1), M.att(START + 2, 2), M.att(START - 1, 3), M.att(START + 1, 0)
    bad = M.att(START + 2, 3, corrupt=True)
    blocks = {"first_middle_last": [[], [a1, a2], [], [a3], []],
              "in_a_row": [[a3], [], [], [], [a1, a2]],
              "only_the_last": [[], [], [], [a1, a2, a3]],
              "invalid_after_empty": [[a4], [], [], [bad, a1], [a2]],
              "empty_after_invalid": [[a4], [a1, bad], [], []]}[shape]
    slots = [START + 4 + k for k in range(len(blocks))]
    M.eng.guard_flags()
    o = both_forms(M, blocks, slots, seed=6)
    assert M.eng.guard_flags() == 0
    want = {"invalid_after_empty": 3, "empty_after_invalid": 1}.get(shape, len(blocks))
    assert o["n_applied"] == want
    for b, blk in enumerate(blocks):
        if not blk:
            assert o["block_status"][b] == (0 if b < want else 2) and o["block_first"][b] == NONE and o["block_reward"][b] == 0
        elif b < want:
            assert o["block_status"][b] == 0 and o["block_reward"][b] > 0


def test_reward_floors_per_attestation(M):
    """three blocks of 40 aggregates (more than a warp's lanes): each block's reward is the sum of its numerators floored one by one,
    and that sum falls short of the floored total by at least 1 gwei; a committee whose members all hold less than one increment sets
    its flags and earns nothing"""
    rng = np.random.default_rng(8)
    B = Batch(M)
    plan = []
    for k in range(3):
        s = START + 4 + k
        picks = [(s - 1 - int(x) // 4, int(x) % 4) for x in rng.choice(4 * SPE, 40, replace=False)]
        if k == 0:
            picks[17] = (START + 3, 0)
        hs = []
        for slot, i in picks:
            bits = rng.random(len(M.committee(slot, i))) < 0.6
            bits[0] = True
            hs.append(B.add(slot, i, bits=None if (slot, i) == (START + 3, 0) else bits.tolist()))
        plan.append(hs)
    wires = B.sign()
    blocks = [[wires[h] for h in p] for p in plan]
    slots = [START + 4 + k for k in range(3)]
    o = both_forms(M, blocks, slots, seed=8)
    assert o["n_applied"] == 3 and not o["status"].any()
    for b in range(3):
        num = [int(x) for x in o["numerator"][40 * b:40 * b + 40]]
        assert int(o["block_reward"][b]) == sum(x // O.DENOMINATOR for x in num) <= sum(num) // O.DENOMINATOR - 1
    low = M.committee(START + 3, 0)
    assert set(low) <= M.low and o["numerator"][17] == 0 and o["flag_mask"][17] == 7
    t = M.tables(8)
    got = M.host(M.args(blocks, slots), t)
    assert all(got[1][v] == 7 for v in low) and any(t[0][v] != 7 for v in low)


# ------------------------------------------------------------------------------------------------ (f): committee sizes
SIZES = [1, 7, 8, 9, 31, 32, 33, 127, 128, 129, 255, 256, 257, 2047, 2048]


@pytest.fixture(scope="module")
def sweep_engine():
    eng = Engine(0)
    yield eng
    eng.close()


@pytest.mark.parametrize("size", SIZES)
def test_committee_size_sweep(sweep_engine, size):
    """every committee of `size` members (one a slot on 4-slot epochs, so they partition the registry), at the tightest bits_stride and
    at 256: first-bit, last-bit, full and alternating bit rows over three blocks, with delays 1-4"""
    W = World(sweep_engine, 4 * size + 5, 4, 5, 1, 1, [size], 256, 12)      # e = 5: slots 20-23; e - 1: 16-19
    first, last, full, alt = [j == 0 for j in range(size)], [j == size - 1 for j in range(size)], None, [j % 2 == 0 for j in range(size)]
    blocks = [[W.att(20, 0, bits=first), W.att(19, 0, bits=last), W.att(18, 0, bits=full), W.att(17, 0, bits=alt)],
              [W.att(21, 0, bits=last), W.att(20, 0, bits=full), W.att(18, 0, bits=alt), W.att(19, 0, bits=first)],
              [W.att(22, 0, bits=full), W.att(21, 0, bits=first), W.att(19, 0, bits=alt), W.att(20, 0, bits=last)]]
    for stride in sorted({(size + 7) // 8, 256}):
        W.stride = stride
        o = both_forms(W, blocks, [21, 22, 23], seed=size)
        assert o["n_applied"] == 3 and not o["status"].any()
        assert o["flag_mask"].tolist() == [7, 3, 2, 2] * 2 + [7, 3, 2, 2]
    # one bit past the committee, at the tight stride: status 8 (3 where the row cannot hold it)
    W.stride = (size + 7) // 8
    o = both_forms(W, [[W.att(22, 0, bits=[True] * (size + 1))]], [23])
    assert o["status"].tolist() == [8 if size % 8 else 3]


# ------------------------------------------------------------------------------------------------ (g): 2^20 validators
def test_full_size_epoch_against_the_oracle():
    """2^20 validators on the mainnet preset (64 committees of 512 a slot, Spec.epoch_committees), 32 blocks of 128 aggregates: block k
    at slot start(e) + k carries the aggregates of every committee of the two slots before it, each with about 95 % of its bits set; the
    call's arguments from Spec.block_attestations_inputs, its outputs and both tables against the oracle"""
    from pos_evolution_b200 import spec as PS
    n, part = 1 << 20, 0.95
    _h = lambda b: hashlib.sha256(b).digest()      # noqa: E731
    eng = Engine(0)
    pspec = PS.Spec(PS.MAINNET, engine=eng)
    p = PS.MAINNET
    H = p.SLOTS_PER_HISTORICAL_ROOT
    sk0 = int.from_bytes(_h(b"full/sk0"), "big") % (R >> 1) or 1
    delta = int.from_bytes(_h(b"full/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), np.uint32).reshape(n, 8)
    pk = eng.sk_to_pk(sk8)
    state = PS.BeaconState(slot=START, fork=PS.Fork(), genesis_validators_root=bytes(32),
                           validators=[PS.Validator(pk[i].tobytes(), 32 * 10**9) for i in range(n)], balances=[32 * 10**9] * n,
                           randao_mixes=[_h(b"mix" + i.to_bytes(8, "little")) for i in range(p.EPOCHS_PER_HISTORICAL_VECTOR)],
                           block_roots=[_h(b"root" + s.to_bytes(8, "little")) for s in range(H)],
                           previous_epoch_participation=[0] * n, current_epoch_participation=[0] * n,
                           previous_justified_checkpoint=PS.Checkpoint(E - 2, _h(b"j-prev")),
                           current_justified_checkpoint=PS.Checkpoint(E - 1, _h(b"j-cur")))
    rng = np.random.default_rng(5)
    committees = {ep: pspec.epoch_committees(state, ep) for ep in (E - 1, E)}
    assert committees[E][2] == 64 and committees[E - 1][2] == 64
    blocks, sks, msgs, sels = [], [], [], []
    for k in range(SPE):
        s = START + k
        atts = []
        for ds in (1, 2):
            slot = s - ds
            ep = slot // SPE
            members, off, cps = committees[ep]
            for i in range(cps):
                c = (slot - ep * SPE) * cps + i
                com = members[off[c]:off[c + 1]]
                bits = rng.random(len(com)) < part
                src = state.current_justified_checkpoint if ep == E else state.previous_justified_checkpoint
                data = PS.AttestationData(slot, i, bytes(state.block_roots[slot % H]), src,
                                          PS.Checkpoint(ep, bytes(state.block_roots[(ep * SPE) % H])))
                sel = com[bits].astype(object)
                sks.append((int(sel.sum()) * delta + len(sel) * sk0) % R)
                msgs.append(pspec.compute_signing_root(data, pspec.get_domain(state, PS.DOMAIN_BEACON_ATTESTER, ep)))
                sels.append(tuple(sorted(int(v) for v in sel)))
                atts.append(PS.Attestation(bits.tolist(), data, None))
        blocks.append(PS.BlockAttestations(s, 0, bytes(state.block_roots[s % H]), atts))
    sigs = eng.sign(np.frombuffer(b"".join(v.to_bytes(32, "little") for v in sks), np.uint32).reshape(-1, 8), np.arange(len(sks), dtype=np.uint32),
                    np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32))
    good = {}
    for j, a in enumerate(a for b in blocks for a in b.attestations):
        a.signature = sigs[j].tobytes()
        good[(sels[j], msgs[j])] = a.signature
    a = pspec.block_attestations_inputs(state, blocks)
    pspec.sync_registry(state)
    t = [(rng.integers(0, 8, n) * (rng.random(n) < 0.3)).astype(np.uint8) for _ in range(2)]
    eng.participation_load(0, t[0])
    eng.participation_load(1, t[1])
    res = eng.block_attestations(**a)
    got = (tuple(res), eng.participation_read(0), eng.participation_read(1))
    o = O.run(a["wire"], a["woff"], a["block_off"], a["block_slot"], a["members"], a["off"], a["cps_prev"], a["cps_cur"],
              a["chain_roots"].reshape(-1, 32), a["justified80"], a["domains64"], SPE, 1, a["bits_stride"], np.full(n, 32 * 10**9, np.uint64),
              a["increment"], a["base_reward_per_increment"], t[0].tolist(), t[1].tolist(),
              lambda idx, root, sig: good.get((tuple(idx), bytes(root))) == bytes(sig))
    same(got, o)
    assert o["n_applied"] == SPE and len(o["status"]) == 4096 and not o["status"].any() and (o["block_reward"] > 0).all()
    eng.close()


# ------------------------------------------------------------------------------------------------ Spec facade on the mainnet preset
def test_spec_mainnet_run_matches_the_spec_block_by_block():
    """Spec.process_block_attestations on the mainnet preset (2 048 validators: one committee of 64 a slot) against
    oracle.spec.process_attestation block by block and against Spec.process_attestations block by block: skipped slots (their roots are
    the previous block's), two blocks of one proposer, an empty block, state.fork.epoch == e with previous_version != current_version
    (previous-epoch attestations sign under the previous version), then the same run whose fourth block holds a previous-epoch
    attestation signed under the current version (status 11)"""
    from oracle import spec as OS
    from pos_evolution_b200 import spec as PS
    n = 2048
    eng = Engine(0)
    pks = [bytes(k) for k in eng.sk_to_pk([scenarios.secret_key(i) for i in range(n)])]
    pspec = PS.Spec(PS.MAINNET, engine=eng)
    ospec = OS.Spec(OS.MAINNET, bls_module=KnownBLS)
    H = OS.MAINNET.SLOTS_PER_HISTORICAL_ROOT
    old, new = bytes.fromhex("00000001"), bytes.fromhex("00000002")
    _, base = scenarios.minimal_state(n, slot=0, preset=OS.MAINNET, pks=pks)

    def proposer(s):
        at = copy.copy(base)
        at.slot = s
        return ospec.get_beacon_proposer_index(at)

    # the first epoch from 3 on with two slots of one proposer after its first slot
    for e in range(3, 40):
        props = {s: proposer(s) for s in range(e * SPE + 1, e * SPE + SPE)}
        twice = [s for s in props if list(props.values()).count(props[s]) > 1]
        if twice:
            break
    start = e * SPE
    pair = [s for s in twice if props[s] == props[twice[0]]][:2]
    slots = sorted({start + 1, start + 2, start + 5, start + 6, start + 9} | set(pair))
    base.slot = slots[0]
    base.fork = OS.Fork(old, new, e)
    base.previous_justified_checkpoint = OS.Checkpoint(e - 2, scenarios._h(b"j-prev"))
    base.current_justified_checkpoint = OS.Checkpoint(e - 1, scenarios._h(b"j-cur"))
    roots = [scenarios._h(b"mainnet run" + s.to_bytes(8, "little")) for s in slots]
    wrong = copy.copy(base)
    wrong.fork = OS.Fork(new, new, 0)

    def root(s):
        return bytes(base.block_roots[s % H]) if s < slots[0] else [r for r, b in zip(roots, slots) if b <= s][-1]

    def att(s, bits=None, under=None):
        E_ = s // SPE
        com = ospec.get_beacon_committee(base, s, 0)
        bits = [True] * len(com) if bits is None else bits
        src = base.current_justified_checkpoint if E_ == e else base.previous_justified_checkpoint
        data = OS.AttestationData(s, 0, root(s), src, OS.Checkpoint(E_, root(E_ * SPE)))
        msg = ospec.compute_signing_root(data, ospec.get_domain(under or base, OS.DOMAIN_BEACON_ATTESTER, E_))
        sel = sorted(set(v for v, b in zip(com, bits) if b))
        sig = bytes(eng.sign([sum(scenarios.secret_key(v) for v in sel) % R], [0], np.frombuffer(msg, np.uint8).reshape(1, 32))[0])
        KnownBLS.good[(tuple(bytes(pks[v]) for v in sel), msg)] = sig
        return OS.Attestation(bits, data, sig)

    def product(a):
        d = a.data
        return PS.Attestation(list(a.aggregation_bits), PS.AttestationData(d.slot, d.index, d.beacon_block_root,
                                                                           PS.Checkpoint(d.source.epoch, d.source.root),
                                                                           PS.Checkpoint(d.target.epoch, d.target.root)), a.signature)

    def advance(st, k):
        if k:
            for t in range(slots[k - 1], slots[k]):
                st.block_roots[t % H] = roots[k - 1]
        st.slot = slots[k]

    def check(blocks):
        st, failed = copy.deepcopy(base), None
        for k in range(len(slots)):
            advance(st, k)
            before = copy.deepcopy(st)
            try:
                for a in blocks[k]:
                    ospec.process_attestation(st, a)
            except AssertionError:
                st, failed = before, k
                break
        proposers = [proposer(s) for s in slots]
        assert len(set(proposers)) < len(proposers)
        ps = TG._pstate(PS, base)
        n_applied, statuses = pspec.process_block_attestations(ps, [PS.BlockAttestations(s, q, r, [product(a) for a in blk])
                                                                    for s, q, r, blk in zip(slots, proposers, roots, blocks)])
        assert n_applied == (len(slots) if failed is None else failed)
        assert ps.balances == st.balances
        assert ps.current_epoch_participation == st.current_epoch_participation
        assert ps.previous_epoch_participation == st.previous_epoch_participation
        # the per-block path on the same blocks
        old_path = TG._pstate(PS, base)
        for k in range(len(slots)):
            advance(old_path, k)
            before = copy.deepcopy(old_path)
            try:
                pspec.process_attestations(old_path, [product(a) for a in blocks[k]])
            except AssertionError:
                old_path = before
                break
        assert old_path.balances == ps.balances
        assert old_path.current_epoch_participation == ps.current_epoch_participation
        assert old_path.previous_epoch_participation == ps.previous_epoch_participation
        return n_applied, statuses, st

    run = []
    for k, s in enumerate(slots):
        half = [j < 32 for j in range(64)]
        blk = [att(s - 1), att(s - 3, bits=half), att(max(start - 1 - k, s - SPE)), att(s - 4, bits=[not b for b in half])]
        run.append([] if k == 2 else blk)
    n_applied, statuses, st = check(run)
    assert n_applied == len(slots) and all(not x.any() for x in statuses) and len(statuses[2]) == 0
    assert any(x != y for x, y in zip(st.previous_epoch_participation, base.previous_epoch_participation))
    run[3] = run[3] + [att(start - 8, under=wrong)]
    n_applied, statuses, _ = check(run)
    assert n_applied == 3 and statuses[3].tolist() == [0, 0, 0, 0, 11]
    eng.close()
