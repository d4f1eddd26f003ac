"""The aggregated-attestation intake at scale and through its consumers, against tests/aggregate_intake_oracle.py:
  - a registry of 2^20 validators, 512 committees of 512 (bits_stride 64), aggregators chosen by their real selection proofs and a planted
    mix (duplicates, subsets, bad aggregates, bad selection proofs, bad outer signatures, non-aggregators, aggregators from the previous
    committee, unknown heads): every output of both ABI forms equals the oracle's;
  - the accepted items, compacted on the device, fed to the block packer give the packer's picks for the oracle's accepted list;
  - Spec.validate_aggregate_and_proofs on a mainnet-preset store (Spec(incremental_tree=True), a fork version that changes between the two
    epochs) equals the oracle over oracle.spec's committees and domains.
Signatures are made on the GPU by Engine.sign over messages the oracle computes; their verdicts are known by construction."""
import hashlib

import numpy as np
import pytest
import torch

import aggregate_intake_oracle as A
import scenarios
from intake_oracle import data128 as make_data
from oracle.bls12_381 import R
from pos_evolution_b200.engine import Engine

pytestmark = pytest.mark.gpu

N_VAL = 1 << 20
SPE, CPS, SIZE, STRIDE, EPOCH = 32, 16, 512, 64, 5
START = EPOCH * SPE
CUR = START + SPE - 1
DOMAINS = bytes([1] * 32) + bytes([5] * 32) + bytes([6] * 32)
# the tree: 0 (slot 0) <- 1 (150) <- 2 (160) <- 3 (170); 4 (165) under 2.  Every head's ancestor at slot 160 is block 2.
PARENT = np.array([0, 0, 1, 2, 2], np.uint32)
SLOT = np.array([0, 150, 160, 170, 165], np.uint64)
ROOTS = np.array([[b + 1] * 32 for b in range(5)], np.uint8)


def _sk(v):
    return (scenarios.SK0 + int(v) * scenarios.SKD) % R


def _sk8(values):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in values), dtype=np.uint32).reshape(-1, 8)


@pytest.fixture(scope="module")
def world():
    eng = Engine(0)
    sk8 = _sk8([_sk(v) for v in range(N_VAL)])
    assert int(eng.registry_load(eng.sk_to_pk(sk8), np.full(N_VAL, 32 * 10**9, np.uint64)).sum()) == N_VAL
    eng.tree_load(PARENT, SLOT, ROOTS, np.ones(5, np.uint8))
    rng = np.random.default_rng(21)
    K = SPE * CPS
    members = rng.permutation(N_VAL)[:K * SIZE].astype(np.uint32)
    off = (np.arange(K + 1) * SIZE).astype(np.uint32)
    slot_msgs = np.frombuffer(b"".join(A.slot_signing_root(START + s, DOMAINS[32:64]) for s in range(SPE)), np.uint8).reshape(SPE, 32)
    proofs = eng.sign(np.ascontiguousarray(sk8[members]), (np.arange(K * SIZE) // (SIZE * CPS)).astype(np.uint32), slot_msgs)
    sel = np.array([A.is_aggregator(SIZE, p.tobytes()) for p in proofs])
    spec = []                                    # (committee, aggregator, bits, data, kind)
    for k in range(K):
        s = START + k // CPS
        heads = [3 if s >= 170 else 2] + ([4] if s >= 165 else [])
        datas = [make_data(s, k % CPS, bytes(ROOTS[h]), EPOCH - 1, bytes(ROOTS[0]), EPOCH, bytes(ROOTS[2])) for h in heads]
        pos = np.flatnonzero(sel[k * SIZE:(k + 1) * SIZE])[:9]
        non = np.flatnonzero(~sel[k * SIZE:(k + 1) * SIZE])
        for p in pos:
            agg, d, r = int(members[k * SIZE + p]), datas[int(rng.integers(len(datas)))], rng.random()
            bits = rng.random(SIZE) < 0.97
            if spec and r < 0.05:
                spec.append(spec[-1][:4] + ("dup",))
            elif r < 0.10 and spec and spec[-1][0] == k:
                spec.append((k, agg, spec[-1][2] & (rng.random(SIZE) < 0.5), spec[-1][3], "ok"))      # a subset after its superset
            elif r < 0.13:
                spec.append((k, agg, bits, d, "agg"))
            elif r < 0.15:
                spec.append((k, agg, bits, d, "sel"))
            elif r < 0.17:
                spec.append((k, agg, bits, d, "sig"))
            elif r < 0.19:
                spec.append((k, int(members[k * SIZE + non[0]]), bits, d, "ok"))                   # not an aggregator
            elif r < 0.21 and k % CPS:
                # an aggregator of the previous committee of the same slot: its proof passes is_aggregator here too; 11 when it was
                # accepted there, 13 otherwise
                prev = np.flatnonzero(sel[(k - 1) * SIZE:k * SIZE])
                spec.append((k, int(members[(k - 1) * SIZE + prev[int(rng.integers(len(prev)))]]), bits, d, "ok"))
            elif r < 0.23:
                spec.append((k, agg, bits, d[:16] + bytes([0xEE] * 32) + d[48:], "ok"))            # an unknown head
            else:
                spec.append((k, agg, bits, d, "ok"))
    n = len(spec)
    assert n >= 4096
    agg_sk, agg_msg = [], []
    for k, agg, bits, d, kind in spec:
        idx = members[k * SIZE:(k + 1) * SIZE][bits].astype(np.int64)
        agg_sk.append((len(idx) * scenarios.SK0 + scenarios.SKD * int(idx.sum())) % R or 1)
        agg_msg.append(bytes(32) if kind == "agg" else A.signing_root(A.data_root(d), DOMAINS[0:32]))
    agg_sig = eng.sign(_sk8(agg_sk), np.arange(n, dtype=np.uint32), np.frombuffer(b"".join(agg_msg), np.uint8).reshape(n, 32))
    pr_msg = np.frombuffer(b"".join(A.slot_signing_root(START + k // CPS, DOMAINS[32:64]) for k, *_ in spec), np.uint8).reshape(n, 32)
    prf = eng.sign(_sk8([_sk(x[1]) for x in spec]), np.arange(n, dtype=np.uint32), pr_msg)
    for i, (k, agg, *_, kind) in enumerate(spec):
        if kind == "sel":      # another aggregator's proof: it passes is_aggregator but not Verify under this aggregator's key
            j = next(j for j in np.flatnonzero(sel[k * SIZE:(k + 1) * SIZE]) if int(members[k * SIZE + j]) != agg)
            prf[i] = proofs[k * SIZE + j]
    aap = [bytes(32) if kind == "sig" else A.aggregate_and_proof_signing_root(agg, bits.tolist(), d, agg_sig[i].tobytes(), prf[i].tobytes(), DOMAINS[64:96])
           for i, (k, agg, bits, d, kind) in enumerate(spec)]
    outer = eng.sign(_sk8([_sk(x[1]) for x in spec]), np.arange(n, dtype=np.uint32), np.frombuffer(b"".join(aap), np.uint8).reshape(n, 32))
    wires = [A.encode(agg, bits.tolist(), d, agg_sig[i].tobytes(), prf[i].tobytes(), outer[i].tobytes()) for i, (k, agg, bits, d, _) in enumerate(spec)]
    ok = [(kind != "sel", kind != "sig", kind != "agg") for *_, kind in spec]
    o = A.validate(wires, members, off, EPOCH, CUR, DOMAINS, CPS, SPE, STRIDE, PARENT, SLOT, ROOTS, lambda i: ok[i])
    return eng, members, off, wires, o


def test_fullsize_registry_against_oracle(world):
    eng, members, off, wires, o = world
    counts = {int(s): int((o.status == s).sum()) for s in np.unique(o.status)}
    assert {0, 10, 11, 12, 13, 14, 15, 16, 17} <= set(counts), counts
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    r = eng.aggregate_and_proof_intake(b"".join(wires), woff, members, off, EPOCH, CUR, DOMAINS, CPS, SPE, STRIDE)
    for f in ("status", "committee", "data_id", "bits", "sigs", "msgs", "target_epoch", "block_idx", "members", "item_off"):
        assert np.array_equal(np.asarray(getattr(r, f)), np.asarray(getattr(o, f))), f
    n = len(wires)
    t = lambda a: torch.from_numpy(np.array(a, copy=True)).cuda()      # noqa: E731
    z = lambda *s, dt=torch.int32: torch.zeros(s, dtype=dt, device="cuda")      # noqa: E731
    d = [z(n), z(n), z(n), z(n, STRIDE, dt=torch.uint8), z(n, 96, dt=torch.uint8), z(n, 32, dt=torch.uint8), z(n, dt=torch.int64), z(n),
         z(n, 8 * STRIDE), z(n + 1)]
    eng.aggregate_and_proof_intake_dev(t(np.frombuffer(b"".join(wires), np.uint8)), t(woff.view(np.int32)), t(members.view(np.int32)),
                                       t(off.view(np.int32)), EPOCH, CUR, DOMAINS, CPS, SPE, *d)
    torch.cuda.synchronize()
    assert np.array_equal(d[0].cpu().numpy(), o.status) and np.array_equal(d[8].cpu().numpy().view(np.uint32), o.members)
    assert np.array_equal(d[3].cpu().numpy(), o.bits) and np.array_equal(d[5].cpu().numpy(), o.msgs)
    assert eng.guard_flags() == 0


def _dense(ids):
    """data ids -> 0 .. k-1 in order of first appearance"""
    _, first, inv = np.unique(ids, return_index=True, return_inverse=True)
    rank = np.argsort(np.argsort(first))
    return rank[inv.reshape(-1)].astype(np.uint32)


def test_accepted_pool_feeds_the_packer(world):
    eng, members, off, wires, o = world
    n = len(wires)
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    t = lambda a: torch.from_numpy(np.array(a, copy=True)).cuda()      # noqa: E731
    z = lambda *s, dt=torch.int32: torch.zeros(s, dtype=dt, device="cuda")      # noqa: E731
    d = [z(n), z(n), z(n), z(n, STRIDE, dt=torch.uint8), z(n, 96, dt=torch.uint8), z(n, 32, dt=torch.uint8), z(n, dt=torch.int64), z(n),
         z(n, 8 * STRIDE), z(n + 1)]
    eng.aggregate_and_proof_intake_dev(t(np.frombuffer(b"".join(wires), np.uint8)), t(woff.view(np.int32)), t(members.view(np.int32)),
                                       t(off.view(np.int32)), EPOCH, CUR, DOMAINS, CPS, SPE, *d)
    keep = torch.nonzero(d[0] == 0).flatten()              # compacted on the device, in list order
    cc, cd = d[1][keep].cpu().numpy().view(np.uint32), d[2][keep].cpu().numpy().view(np.uint32)
    bits, sigs = d[3][keep].cpu().numpy(), d[4][keep].cpu().numpy()
    acc = np.flatnonzero(o.status == 0)
    table = np.zeros(SPE * CPS, np.uint8)
    args = (10**9, 64)
    got = eng.pack_attestations(members, off, table, cc, _dense(cd), np.full(len(cc), 7, np.uint8), bits, sigs, 128, *args)
    want = eng.pack_attestations(members, off, table, o.committee[acc], _dense(o.data_id[acc]), np.full(len(acc), 7, np.uint8), o.bits[acc],
                                 o.sigs[acc], 128, *args)
    assert len(want.committee) == 128
    for f in want._fields:
        assert np.array_equal(getattr(got, f), getattr(want, f)), f


def test_spec_facade_on_mainnet_store():
    from oracle import spec as OS
    from pos_evolution_b200 import spec as PS
    n_val, cur = 2048, 70                                   # mainnet: one committee of 64 per slot; epochs 2 and 1 are open
    eng = Engine(0)
    sks = [scenarios.secret_key(i) for i in range(n_val)]
    pks = [bytes(p) for p in eng.sk_to_pk(sks)]
    ospec, ostate = scenarios.minimal_state(n_val, cur, preset=OS.MAINNET, pks=pks)
    ostate.fork = OS.Fork(bytes(4), bytes.fromhex("00000001"), 2)      # epoch 1 signs with the previous version, epoch 2 with the current one
    state = PS.BeaconState(slot=cur, fork=PS.Fork(bytes(4), bytes.fromhex("00000001"), 2), genesis_validators_root=ostate.genesis_validators_root,
                           validators=[PS.Validator(v.pubkey, v.effective_balance) for v in ostate.validators], balances=list(ostate.balances),
                           randao_mixes=list(ostate.randao_mixes), block_roots=list(ostate.block_roots),
                           previous_epoch_participation=[0] * n_val, current_epoch_participation=[0] * n_val)
    # store.blocks: a chain 0 .. 64 .. 68 and a fork at 65; finalized and justified at the first block
    bslot = [0, 10, 31, 32, 40, 63, 64, 66, 68, 65]
    bparent = [0, 0, 1, 2, 3, 4, 5, 6, 7, 6]
    roots = [hashlib.sha256(b"agg-block%d" % b).digest() for b in range(len(bslot))]
    cp = PS.Checkpoint(0, roots[0])
    state.current_justified_checkpoint = state.finalized_checkpoint = cp
    store = PS.Store(cur * 12, 0, cp, cp, cp, PS.ZERO32, set())
    for b in range(len(bslot)):
        store.blocks[roots[b]] = PS.BeaconBlock(bslot[b], roots[bparent[b]] if b else bytes(32))
        store.block_states[roots[b]] = state
    store.checkpoint_states[cp] = state
    sp = PS.Spec(PS.MAINNET, engine=eng, incremental_tree=True)
    anc = lambda b, s: anc(bparent[b], s) if bslot[b] > s else b      # noqa: E731
    rng = np.random.default_rng(8)
    dom = lambda t, e: ospec.get_domain(ostate, t, e)      # noqa: E731
    plan = []                                              # (slot, head block, aggregator position, kind)
    for s in list(range(38, 71, 3)) + [5, 71]:
        e = s // 32
        heads = [b for b in range(len(bslot)) if bslot[b] <= s and b != 0] or [0]
        for _ in range(3):
            plan.append((s, heads[int(rng.integers(len(heads)))], rng.random()))
    items, ok = [], []
    for s, h, r in plan:
        e = s // 32
        com = ospec.get_beacon_committee(ostate, s, 0)
        sel_dom, aap_dom = dom(A.DOMAIN_SELECTION_PROOF, e), dom(A.DOMAIN_AGGREGATE_AND_PROOF, e)
        proofs = [bytes(p) for p in eng.sign([sks[v] for v in com], [0] * len(com),
                                             np.frombuffer(A.slot_signing_root(s, sel_dom), np.uint8).reshape(1, 32))]
        aggp = [j for j in range(len(com)) if A.is_aggregator(len(com), proofs[j])]
        j = aggp[int(rng.integers(len(aggp)))] if r < 0.9 else int(np.flatnonzero([not A.is_aggregator(len(com), p) for p in proofs])[0])
        bits = [bool(x) for x in rng.random(len(com)) < 0.9]
        data = PS.AttestationData(s, 0, roots[h], PS.Checkpoint(e - 1 if e else 0, roots[0]), PS.Checkpoint(e, roots[anc(h, 32 * e)]))
        msg = A.signing_root(A.data_root(PS.serialize_attestation_data(data)), dom(OS.DOMAIN_BEACON_ATTESTER, e))
        bad = r > 0.8 and r < 0.9
        asig = bytes(eng.sign([sum(sks[com[i]] for i in range(len(com)) if bits[i]) % R], [0],
                              np.frombuffer(bytes(32) if bad else msg, np.uint8).reshape(1, 32))[0])
        m = PS.AggregateAndProof(com[j], PS.Attestation(bits, data, asig), proofs[j])
        osig = bytes(eng.sign([sks[com[j]]], [0], np.frombuffer(A.aggregate_and_proof_signing_root(
            com[j], bits, PS.serialize_attestation_data(data), asig, proofs[j], aap_dom), np.uint8).reshape(1, 32))[0])
        items.append(PS.SignedAggregateAndProof(m, osig))
        ok.append((True, True, not bad))
    status, accepted = sp.validate_aggregate_and_proofs(state, store, items, current_slot=cur)
    # the oracle: one call per open epoch over oracle.spec's committees and domains, the store's blocks as the tree
    want = [7] * len(items)
    tparent, tslot, troots = np.array(bparent, np.uint32), np.array(bslot, np.uint64), np.frombuffer(b"".join(roots), np.uint8).reshape(-1, 32)
    for e in (2, 1):
        sel = [i for i, x in enumerate(items) if x.message.aggregate.data.slot // 32 == e]
        coms = [ospec.get_beacon_committee(ostate, s, 0) for s in range(32 * e, 32 * e + 32)]
        members = np.concatenate([np.array(c, np.uint32) for c in coms])
        off = np.concatenate([[0], np.cumsum([len(c) for c in coms])]).astype(np.uint32)
        domains = b"".join(dom(t, e) for t in (OS.DOMAIN_BEACON_ATTESTER, A.DOMAIN_SELECTION_PROOF, A.DOMAIN_AGGREGATE_AND_PROOF))
        o = A.validate([PS.serialize_signed_aggregate_and_proof(items[i]) for i in sel], members, off, e, cur, domains, 1, 32,
                       (max(len(c) for c in coms) + 7) // 8, tparent, tslot, troots, lambda k: ok[sel[k]])
        for k, i in enumerate(sel):
            want[i] = int(o.status[k])
    assert status == want
    assert 0 in want and 7 in want and (12 in want or 16 in want), sorted(set(want))
    assert accepted == [items[i].message.aggregate for i in range(len(items)) if want[i] == 0]
