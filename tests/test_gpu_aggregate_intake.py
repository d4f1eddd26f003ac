"""The aggregated-attestation intake on the GPU (b2_aggregate_and_proof_intake / _dev, Engine.aggregate_and_proof_intake / _dev) against
tests/aggregate_intake_oracle.py: every status 0-20 and every output on small ragged committees, both ABI forms, on_attestation of the
accepted aggregates through latest_messages_update_dev, the device guards and the host form's refusals.  Signatures are made on the
GPU by b2_sign over messages the oracle computes; their verdicts are known by construction (the right key over the right message, or a
planted corruption)."""
import numpy as np
import pytest
import torch

import aggregate_intake_oracle as A
from intake_oracle import data128 as make_data
from oracle.bls12_381 import R
from pos_evolution_b200._lib import B2Error
from pos_evolution_b200.engine import Engine

pytestmark = pytest.mark.gpu

SPE, CPS, STRIDE, TARGET, RANGE = 4, 2, 4, 8, 32
EPOCH, CUR = 3, 14                               # slots 12 .. 15 of epoch 3; the current slot is 14
SIZES = [17, 20, 24, 31, 9, 12, 3, 5]            # committees 0-3: modulo 2-3 at TARGET 8; 4-7: modulo 1
N_VAL = 160
DOMAINS = bytes([1] * 32) + bytes([5] * 32) + bytes([6] * 32)
# the tree: 0 (slot 0) <- 1 (5) <- 2 (11) <- 3 (12) <- 4 (13); 5 (12) under 2
PARENT = np.array([0, 0, 1, 2, 3, 2], np.uint32)
SLOT = np.array([0, 5, 11, 12, 13, 12], np.uint64)
ROOTS = np.array([[b + 1] * 32 for b in range(6)], np.uint8)


@pytest.fixture(scope="module")
def env():
    eng = Engine(0)
    sks = list(range(1, N_VAL + 1))
    pks = eng.sk_to_pk(sks)
    eng.registry_load(pks, np.full(N_VAL, 32 * 10**9, np.uint64))
    eng.tree_load(PARENT, SLOT, ROOTS, np.ones(6, np.uint8))
    rng = np.random.default_rng(11)
    members = rng.permutation(N_VAL)[:sum(SIZES)].astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(SIZES)]).astype(np.uint32)
    return eng, sks, members, off


def _committee(members, off, c):
    return [int(x) for x in members[off[c]:off[c + 1]]]


class Builder:
    """Items signed on the GPU in two rounds (selection proofs and aggregates, then the outer signatures)."""

    def __init__(self, eng, sks, members, off):
        self.eng, self.sks, self.members, self.off = eng, sks, members, off
        self.specs = []

    def proof(self, v, slot):
        m = np.frombuffer(A.slot_signing_root(slot, DOMAINS[32:64]), np.uint8).reshape(1, 32)
        return bytes(self.eng.sign([self.sks[v]], [0], m)[0])

    def aggregator(self, c, ok=True, skip=()):
        """a member of committee c whose selection proof passes is_aggregator (ok) or fails it"""
        slot = 12 + c // CPS
        com = _committee(self.members, self.off, c)
        for v in com:
            if v not in skip and A.is_aggregator(len(com), self.proof(v, slot), TARGET) == ok:
                return v
        raise AssertionError("no such member")

    def add(self, c, bits, agg, head=None, target=3, slot=None, index=None, tepoch=None, corrupt=None, head_root=None, target_root=None):
        slot = 12 + c // CPS if slot is None else slot
        head = (3 if slot == 12 else 4) if head is None else head      # a head at or below data.slot whose ancestor at slot 12 is block 3
        d = make_data(slot, c % CPS if index is None else index, bytes(ROOTS[head]) if head_root is None else head_root, 2, bytes(32),
                      slot // SPE if tepoch is None else tepoch, bytes(ROOTS[target]) if target_root is None else target_root)
        self.specs.append(dict(c=c, bits=list(bits), agg=agg, d=d, slot=slot, corrupt=corrupt))
        return len(self.specs) - 1

    def build(self):
        wires, ok = [], []
        for s in self.specs:
            com = _committee(self.members, self.off, s["c"]) if s["c"] < len(SIZES) else []
            sel = [com[j] for j, b in enumerate(s["bits"]) if b and j < len(com)]
            msg = A.signing_root(A.data_root(s["d"]), DOMAINS[0:32])
            if s["corrupt"] == "agg":
                msg = bytes(32)
            sk = sum(self.sks[v] for v in sel) % R or 1
            s["agg_sig"] = bytes(self.eng.sign([sk], [0], np.frombuffer(msg, np.uint8).reshape(1, 32))[0])
            v = s["agg"] if s["agg"] < N_VAL else 0
            s["proof"] = self.proof(v, s["slot"] + (1 if s["corrupt"] == "sel" else 0))
        for s in self.specs:
            m = A.aggregate_and_proof_signing_root(s["agg"], s["bits"], s["d"], s["agg_sig"], s["proof"], DOMAINS[64:96])
            if s["corrupt"] == "sig":
                m = bytes(32)
            v = s["agg"] if s["agg"] < N_VAL else 0
            sig = bytes(self.eng.sign([self.sks[v]], [0], np.frombuffer(m, np.uint8).reshape(1, 32))[0])
            wires.append(A.encode(s["agg"], s["bits"], s["d"], s["agg_sig"], s["proof"], sig))
            ok.append((s["corrupt"] != "sel", s["corrupt"] != "sig", s["corrupt"] != "agg"))
        return wires, ok


def _scenario(env):
    eng, sks, members, off = env
    b = Builder(eng, sks, members, off)
    full = lambda c: [True] * SIZES[c]                                      # noqa: E731
    half = lambda c: [j < SIZES[c] // 2 for j in range(SIZES[c])]          # noqa: E731
    rest = lambda c: [j >= SIZES[c] // 2 for j in range(SIZES[c])]         # noqa: E731
    a0, a1, a4 = b.aggregator(0), b.aggregator(1), b.aggregator(4)
    a0b = b.aggregator(0, skip=(a0,))
    c5, c6 = _committee(members, off, 5), _committee(members, off, 6)
    b.add(0, half(0), a0)                                 # 0 accept
    b.add(0, half(0)[:-1] + [False], a0b)                 # 10 subset of an accepted item
    b.add(0, rest(0), a0)                                 # 11 same aggregator
    b.add(0, rest(0), a0b)                                # 0 disjoint bits of the same data
    b.add(1, full(1), a1, corrupt="agg")                  # 16
    b.add(4, full(4), a1)                                 # 13: a1 is not in committee 4 and is accepted only later
    b.add(1, full(1), a1)                                 # 0: the failed duplicate does not shadow it
    b.add(4, full(4), a0)                                 # 11: aggregator a0 was accepted in committee 0
    b.add(4, full(4), a1)                                 # 11: a1 was accepted in committee 1
    b.add(5, full(5), c6[0])                              # 13: not in the committee, never accepted
    b.add(0, full(0), b.aggregator(0, ok=False))          # 12
    b.add(4, full(4), a4, corrupt="sel")                  # 14
    b.add(5, full(5), c5[0], corrupt="sig")               # 15
    b.add(5, full(5), c5[1], head_root=bytes([0xAB] * 32))          # 17
    b.add(2, full(2), b.aggregator(2), target_root=bytes([0xAC] * 32))      # 18
    b.add(1, full(1), b.aggregator(1, skip=(a1,)), head=4)          # 19: the head's slot 13 > data.slot 12
    b.add(3, full(3), b.aggregator(3), head=4, target=5)            # 20: block 5 is not the ancestor at slot 12
    b.add(4, full(4), a4, slot=15, index=0)               # 5: slot 15 > the current slot
    b.add(4, full(4), a4, index=2)                        # 4
    b.add(4, full(4), a4, tepoch=2)                       # 6
    b.add(4, full(4), a4, slot=10, index=0, head=2, target=2)      # 7: epoch 2
    b.add(4, full(4) + [True], a4)                        # 8
    b.add(4, [False] * SIZES[4], a4)                      # 9
    b.add(4, [True] * (8 * STRIDE + 1), a4)               # 3
    b.add(5, full(5), c5[2])                              # 0: the item with status 15 of the same data does not shadow it
    wires, ok = b.build()
    wires.append(wires[0][:150])                          # 1: truncated
    w = bytearray(wires[1])
    w[-1] = 0
    wires.append(bytes(w))                                # 2: no delimiter
    ok += [(True, True, True)] * 2
    return wires, ok


def _host_call(eng, members, off, wires, epoch=EPOCH, cur=CUR):
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    return eng.aggregate_and_proof_intake(b"".join(wires), woff, members, off, epoch, cur, DOMAINS, CPS, SPE, STRIDE, TARGET, RANGE)


def _oracle(members, off, wires, ok):
    return A.validate(wires, members, off, EPOCH, CUR, DOMAINS, CPS, SPE, STRIDE, PARENT, SLOT, ROOTS, lambda i: ok[i], TARGET, RANGE)


def _same(r, o):
    for f in ("status", "committee", "data_id", "bits", "sigs", "msgs", "target_epoch", "block_idx", "members", "item_off"):
        assert np.array_equal(np.asarray(getattr(r, f)), np.asarray(getattr(o, f))), f


def _dev_call(eng, members, off, wires, woff=None, d_off=None):
    n = len(wires)
    if woff is None:
        woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    t = lambda a: torch.from_numpy(np.array(a, copy=True)).cuda()      # noqa: E731
    d = dict(status=torch.zeros(n, dtype=torch.int32), committee=torch.zeros(n, dtype=torch.int32), data_id=torch.zeros(n, dtype=torch.int32),
             bits=torch.zeros((n, STRIDE), dtype=torch.uint8), sigs=torch.zeros((n, 96), dtype=torch.uint8),
             msgs=torch.zeros((n, 32), dtype=torch.uint8), target_epoch=torch.zeros(n, dtype=torch.int64),
             block_idx=torch.zeros(n, dtype=torch.int32), members=torch.zeros((n, 8 * STRIDE), dtype=torch.int32),
             item_off=torch.zeros(n + 1, dtype=torch.int32))
    d = {k: v.cuda() for k, v in d.items()}
    d_members, d_off_t = t(members.view(np.int32)), t((off if d_off is None else d_off).astype(np.uint32).view(np.int32))
    eng.aggregate_and_proof_intake_dev(t(np.frombuffer(b"".join(wires), np.uint8)), t(woff.view(np.int32)), d_members, d_off_t, EPOCH, CUR, DOMAINS,
                                       CPS, SPE, d["status"], d["committee"], d["data_id"], d["bits"], d["sigs"], d["msgs"], d["target_epoch"],
                                       d["block_idx"], d["members"], d["item_off"], TARGET, RANGE)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in d.items()}
    for k in ("committee", "data_id", "block_idx", "members", "item_off"):
        out[k] = out[k].view(np.uint32)
    out["target_epoch"] = out["target_epoch"].view(np.uint64)
    return type("R", (), out)(), d


def test_every_status_against_oracle(env):
    eng, sks, members, off = env
    wires, ok = _scenario(env)
    o = _oracle(members, off, wires, ok)
    assert set(o.status.tolist()) == set(range(21)), sorted(set(range(21)) - set(o.status.tolist()))
    few = _oracle(members, off, wires[:3], ok[:3])
    _same(_dev_call(eng, members, off, wires[:3])[0], few)
    r = _host_call(eng, members, off, wires)
    _same(r, o)
    rd, _ = _dev_call(eng, members, off, wires)
    _same(rd, o)
    # the short list again, on the scratch the full one grew
    _same(_dev_call(eng, members, off, wires[:3])[0], few)
    assert eng.guard_flags() == 0


def test_construction_matches_oracle_bls(env):
    """the verdicts the scenario assumes by construction, for one honest item and each planted corruption, from oracle.bls_sig"""
    from oracle import bls_sig as OB
    eng, sks, members, off = env
    wires, ok = _scenario(env)
    seen = set()
    for i, w in enumerate(wires):
        st, f = A.decode(w, 8 * STRIDE)
        if st or ok[i] in seen:
            continue
        agg, bits, d, agg_sig, proof, sig = f
        c = (int.from_bytes(d[0:8], "little") - 12) * CPS + int.from_bytes(d[8:16], "little")
        if not 0 <= c < 6 or agg >= N_VAL or len(bits) != SIZES[c]:
            continue
        seen.add(ok[i])
        pk = OB.SkToPk(sks[agg])
        slot = int.from_bytes(d[0:8], "little")
        sel_ok = OB.Verify(pk, A.slot_signing_root(slot, DOMAINS[32:64]), proof)
        sig_ok = OB.Verify(pk, A.aggregate_and_proof_signing_root(agg, bits, d, agg_sig, proof, DOMAINS[64:96]), sig)
        com = _committee(members, off, c)
        fav_ok = OB.FastAggregateVerify([OB.SkToPk(sks[com[j]]) for j, b in enumerate(bits) if b], A.signing_root(A.data_root(d), DOMAINS[0:32]), agg_sig)
        assert (sel_ok, sig_ok, fav_ok) == ok[i], i
    assert len(seen) == 4


def test_accepted_rows_feed_on_attestation(env):
    eng, sks, members, off = env
    wires, ok = _scenario(env)
    o = _oracle(members, off, wires, ok)
    eng.latest_messages_reset()
    _, d = _dev_call(eng, members, off, wires)
    accept = (d["status"] == 0).to(torch.uint8)
    eng.latest_messages_update_dev(d["members"], d["item_off"], d["bits"], d["target_epoch"], d["block_idx"], accept)
    torch.cuda.synchronize()
    epoch, blk, has = eng.latest_messages_read()
    want = {}
    for i in np.flatnonzero(o.status == 0):                # on_attestation of the accepted aggregates, in list order
        com = _committee(members, off, int(o.committee[i]))
        for j, v in enumerate(com):
            if (o.bits[i, j >> 3] >> (j & 7)) & 1 and (v not in want or int(o.target_epoch[i]) > want[v][0]):
                want[v] = (int(o.target_epoch[i]), int(o.block_idx[i]))
    assert want and {int(v) for v in np.flatnonzero(has)} == set(want)
    for v, (e, b) in want.items():
        assert (int(epoch[v]), int(blk[v])) == (e, b)
    eng.latest_messages_reset()


def test_device_guards(env):
    eng, sks, members, off = env
    wires, ok = _scenario(env)
    eng.guard_flags()
    n = len(wires)
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    bad = woff.copy()
    bad[3] = bad[2] - 1                                    # item 2 reversed; item 3 then starts before it ends
    r, _ = _dev_call(eng, members, off, wires, woff=bad)
    assert r.status[2] == 1 and eng.guard_flags() & 2
    o = _oracle(members, off, wires, ok)
    # a committee row that ends past the members: its items read status 8, nothing past the array is read
    d_off = off.copy()
    d_off[5:] = np.uint32(10**6)
    r, _ = _dev_call(eng, members, off, wires, d_off=d_off)
    c4 = [i for i in range(n) if o.committee[i] == 4]
    assert c4 and all(int(r.status[i]) == 8 for i in c4) and eng.guard_flags() & 2
    # an aggregator index far outside the registry: not a member (13), the registry is never read for it
    b = Builder(eng, sks, members, off)
    b.add(4, [True] * SIZES[4], 2**40)
    w2, _ = b.build()
    r, _ = _dev_call(eng, members, off, w2)
    assert r.status.tolist() == [13] and eng.guard_flags() == 0
    # a member index outside the registry that is the aggregator: check 14 fails it and records the bad index
    mem = members.copy()
    mem[off[4]] = 10**7
    b = Builder(eng, sks, mem, off)
    b.add(4, [False] + [True] * (SIZES[4] - 1), 10**7)
    w3, _ = b.build()
    r, _ = _dev_call(eng, mem, off, w3)
    assert r.status.tolist() == [14] and eng.guard_flags() & 1


def test_refused_host_calls_change_nothing(env):
    eng, sks, members, off = env
    wires, ok = _scenario(env)
    first = _host_call(eng, members, off, wires)
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    wire = b"".join(wires)
    bad_woff = woff.copy()
    bad_woff[-1] += 1
    bad_off = off.copy()
    bad_off[1] = 40                                        # a committee of 40 > 8 * STRIDE
    calls = [dict(woff=bad_woff), dict(off=bad_off), dict(epoch=1), dict(epoch=5), dict(stride=0), dict(stride=257), dict(target=0),
             dict(cps=3)]
    for kw in calls:
        with pytest.raises(B2Error):
            eng.aggregate_and_proof_intake(wire, kw.get("woff", woff), members, kw.get("off", off), kw.get("epoch", EPOCH), CUR, DOMAINS,
                                           kw.get("cps", CPS), SPE, kw.get("stride", STRIDE), kw.get("target", TARGET), RANGE)
    again = _host_call(eng, members, off, wires)
    for f in first._fields:
        assert np.array_equal(getattr(first, f), getattr(again, f)), f
    fresh = Engine(0)
    with pytest.raises(B2Error):                           # no registry, no tree
        _host_call(fresh, members, off, wires)
    fresh.close()
