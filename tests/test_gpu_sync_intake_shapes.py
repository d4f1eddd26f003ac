"""The two sync intakes (b2_sync_committee_messages and b2_sync_contribution_and_proof_intake, both ABI forms; kernels in csrc/syncmsg.cuh and
csrc/synccontrib.cuh) outside the 4-subnet preset shapes, compared byte for byte with tests/sync_messages_oracle.py and
tests/sync_contributions_oracle.py:
  * every committee shape class the ABI takes: subcommittees of 1, 9, 40, 125, 510, 260, 768 and 1 024 positions (padding bits, a partial
    last word of check 8, Bitvector roots of 1-4 chunks), aggregator moduli 1, 3, 7, 8, 64 and 341;
  * distinct roots on one home slot of the root tables (tests/sync_keys.py), probes that wrap past the last slot, byte-equal copies behind
    a chain, a root first entered by an item that later fails;
  * more than one CTA of roots: leaders past list index 1 024, 1 024 roots, ties of `best` in different CTAs;
  * u64 fields with a nonzero high word;
  * the exceptional additions of the signature sums (P + P, P + (-P), a committee of one validator, sums at infinity);
  * the rows past n_roots of both forms;
  * one engine running messages, contributions and b2_aggregate_verify interleaved, against fresh engines.
Signatures come from Engine.sign (secret key v + 1; the last validator holds r - 1, the negation of validator 0's key) and the oracles'
verdicts from the known signers (their closed-form mode), except where a case says it checks real signatures.
Run on an H100:
    python -m pytest tests/test_gpu_sync_intake_shapes.py -m gpu -s"""
import ctypes
import time

import numpy as np
import pytest
import torch

import sync_contributions_oracle as C
import sync_keys as K
import sync_messages_oracle as M
import sync_oracle as SO
from oracle.bls12_381 import R
from pos_evolution_b200.engine import Engine, SyncContributionsResult, SyncMessagesResult

pytestmark = pytest.mark.gpu

N_VAL, SLOT = 4096, 1234567
U64 = (1 << 64) - 1
DOM = bytes([7]) + bytes(range(31))                                   # the sync committee domain
DOMS = DOM + bytes([8]) + bytes(range(31)) + bytes([9]) + bytes(range(31))
SENTINEL = 0xA5
INF = bytes([0xC0]) + bytes(95)


def sk(v: int) -> int:
    return R - 1 if v == N_VAL - 1 else int(v) + 1


@pytest.fixture(scope="module")
def env():
    eng = Engine(0)
    pks = eng.sk_to_pk([sk(v) for v in range(N_VAL)])
    eng.registry_load(pks, np.full(N_VAL, 32 * 10**9, np.uint64))
    yield eng, pks
    eng.close()


def _fresh(pks):
    e = Engine(0)
    e.registry_load(pks, np.full(N_VAL, 32 * 10**9, np.uint64))
    return e


def _sign(eng, keys, msgs):
    """Engine.sign of one (key, message) per entry, one call; a zero key gives the point at infinity"""
    keys = [int(k) % R for k in keys]
    live = [i for i, k in enumerate(keys) if k]
    out = [INF] * len(keys)
    if live:
        uniq = sorted({msgs[i] for i in live})
        at = {m: j for j, m in enumerate(uniq)}
        s = eng.sign([keys[i] for i in live], np.array([at[msgs[i]] for i in live], np.uint32),
                     np.frombuffer(b"".join(uniq), np.uint8).reshape(-1, 32))
        for j, i in enumerate(live):
            out[i] = s[j].tobytes()
    return out


def _woff(wires):
    return np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)


def _timed(name, t0):
    print("\n%s: %.1f s wall on %s" % (name, time.perf_counter() - t0, torch.cuda.get_device_name(0)))


# ------------------------------------------------------------------------------------------------------------ messages

def _msg_wires(eng, items, dom=DOM):
    """items: (slot, root, validator_index u64, signing key or None for the validator's own) -> wires"""
    keys = [(sk(v) if v < N_VAL else 1) if k is None else k for _, _, v, k in items]
    sigs = _sign(eng, keys, [M.signing_root(r, dom) for _, r, _, _ in items])
    return [M.encode(s, r, v, sig) for (s, r, v, _), sig in zip(items, sigs)]


def _msg_expect(eng, items, wires, subnets, pv, count, current_slot, dom=DOM):
    good = [v < N_VAL and (k is None or k % R == sk(v) % R) for _, _, v, k in items]
    want = M.validate(wires, subnets, [int(x) for x in pv], N_VAL, lambda v: None, current_slot, dom, count=count,
                      verify=lambda a, pk, m, s: good[a], secret_key=sk, closed_form=True)
    return M.sign_closed_form(want, lambda ks, ms: _sign(eng, ks, ms))


def _msg_arrays(r, size, count):
    sub = size // count
    k = len(r.roots)
    cb, cs, cp = np.zeros((k, count, (sub + 7) // 8), np.uint8), np.zeros((k, count, 96), np.uint8), np.zeros((k, count), np.uint8)
    ab, asig = np.zeros((k, (size + 7) // 8), np.uint8), np.zeros((k, 96), np.uint8)
    for (j, s), c in r.contributions.items():
        cb[j, s] = np.frombuffer(M.pack(c.aggregation_bits), np.uint8)
        cs[j, s] = np.frombuffer(c.signature, np.uint8)
        cp[j, s] = 1
    for j, a in enumerate(r.aggregates):
        ab[j] = np.frombuffer(M.pack(a.sync_committee_bits), np.uint8)
        asig[j] = np.frombuffer(a.sync_committee_signature, np.uint8)
    roots = np.frombuffer(b"".join(r.roots), np.uint8).reshape(k, 32) if k else np.zeros((0, 32), np.uint8)
    return (np.array(r.status, np.int32), np.array(r.root_id, np.uint32), roots, cb, cs, cp, ab, asig)


def _assert_equal(got, want, names):
    for name, g, w in zip(names, got, want):
        g = np.asarray(g)
        assert g.shape == w.shape and np.array_equal(g.astype(w.dtype), w), name


MSG_NAMES = ("status", "root_id", "roots", "contrib_bits", "contrib_sigs", "contrib_present", "agg_bits", "agg_sigs")
SCC_NAMES = ("status", "root_id", "roots", "best", "agg_bits", "agg_sigs")


def _t(a):
    a = np.asarray(a)
    return torch.as_tensor(a.astype(np.int32) if a.dtype == np.uint32 else a.copy(), device=torch.device("cuda", 0))


def _msg_dev(eng, wires, subnets, pv, count, slot):
    wire = np.frombuffer(b"".join(wires), np.uint8)
    r = eng.sync_committee_messages_dev(_t(wire), _t(_woff(wires)), _t(np.asarray(subnets, np.uint32)), _t(np.asarray(pv, np.uint32)), count,
                                        slot, DOM)
    torch.cuda.synchronize()
    out = [x.cpu().numpy() for x in r]
    out[1] = out[1].view(np.uint32)
    return out


def _msg_run(eng, wires, subnets, pv, count, slot, want):
    """both forms against the oracle's arrays; returns the host form's result"""
    w = _msg_arrays(want, len(pv), count)
    host = eng.sync_committee_messages(b"".join(wires), _woff(wires), subnets, pv, count, slot, DOM)
    _assert_equal(host, w, MSG_NAMES)
    _assert_equal(_msg_dev(eng, wires, subnets, pv, count, slot), w, MSG_NAMES)
    return host


def _verify_aggregates(eng, pks, pv, roots, agg_bits, agg_sigs, dom=DOM):
    """each produced SyncAggregate through b2_sync_committee_load(size) and b2_sync_aggregate_verify"""
    if not len(roots):
        return
    eng.sync_committee_load(pks[np.asarray(pv, np.int64)], len(pv))
    msgs = np.frombuffer(b"".join(M.signing_root(r, dom) for r in roots), np.uint8).reshape(-1, 32)
    assert eng.sync_aggregate_verify(np.zeros(len(roots), np.uint32), agg_bits, msgs, agg_sigs).tolist() == [1] * len(roots)


# (committee_size, subnet_count, target_aggregators) -> sub and the aggregator modulus max(1, sub // target)
SHAPES = [(1, 1, 5), (7, 7, 1), (36, 4, 3), (40, 1, 41), (512, 4, 16), (1000, 8, 17), (1020, 2, 70), (780, 3, 80), (768, 1, 12),
          (1024, 1, 3), (1024, 4, 32), (1024, 8, 16)]


def _committee(size, rng):
    return rng.permutation(N_VAL - 1)[:size].astype(np.uint32)      # the negated key stays out


@pytest.mark.parametrize("size,count,target", SHAPES, ids=["%dx%d" % s[:2] for s in SHAPES])
def test_message_shapes(env, size, count, target):
    """per subnet: members sign root A, the subnet's last position alone signs root B (a row with only bit sub - 1), bad signatures
    before good ones, duplicates, another slot, a validator outside the registry, a subnet of another member and one >= count"""
    eng, pks = env
    t0 = time.perf_counter()
    rng = np.random.default_rng(size * 31 + count)
    sub = size // count
    pv = _committee(size, rng)
    ra, rb = bytes([0x10 + count]) * 32, bytes([0x20 + count]) * 32
    items, subnets = [], []

    def add(item, s):
        items.append(item)
        subnets.append(s)

    for s in range(count):
        add((SLOT, ra, int(pv[s * sub]), sk(int(pv[s * sub])) + 1), s)        # 6, before the first position's good message
        ps = list(range(s * sub, (s + 1) * sub))
        if sub > 48:
            ps = sorted(set([ps[0], ps[-1]] + list(rng.choice(ps, 46, replace=False))))
        for j, p in enumerate(ps):
            v, last = int(pv[p]), p == (s + 1) * sub - 1
            if j % 7 == 3:
                add((SLOT, ra, v, sk(v) + 1), s)                             # 6, then the good one
            add((SLOT, rb if last else ra, v, None), s)
            if j % 11 == 5:
                add((SLOT, ra, v, None), s)                                  # 5
        v = int(pv[s * sub])
        add((SLOT + 1, ra, v, None), s)                                      # 2
        add((SLOT, ra, N_VAL + s, None), s)                                  # 3
        add((SLOT, ra, v, None), count)                                      # 4: subnet >= count
        if count > 1:
            add((SLOT, ra, int(pv[((s + 1) % count) * sub]), None), s)       # 4: another subnet's member
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, subnets, pv, count, SLOT)
    assert {0, 2, 3, 4, 6} <= set(want.status) and (5 in want.status or sub < 6)
    assert want.roots == [ra, rb] or (sub == 1 and want.roots == [rb])
    for s in range(count):      # root B's row on every subnet is bit sub - 1 alone
        rbi = want.roots.index(rb)
        assert want.contributions[(rbi, s)].aggregation_bits == [False] * (sub - 1) + [True]
    host = _msg_run(eng, wires, subnets, pv, count, SLOT, want)
    _verify_aggregates(eng, pks, pv, want.roots, host.agg_bits, host.agg_sigs)
    _timed("messages %dx%d, %d items" % (size, count, len(wires)), t0)


# ------------------------------------------------------------------------------------------------------------ contributions

def _proofs(eng, vs, subnets, slot=SLOT, doms=DOMS):
    return _sign(eng, [sk(v) for v in vs], [C.signing_root(C.selection_data_root(slot, s), doms[32:64]) for s in subnets])


def _scc_wires(eng, plan, pv, sub, count, doms=DOMS):
    """plan: dicts with g (aggregator, u64), s (subcommittee_index field, u64), root, bits (bool list, may run into the padding), and
    optional slot, proof (bytes), bad (a set of 'proof', 'outer', 'sig': that signature is made with the key + 1) -> wires, signed in
    three Engine.sign calls"""
    slot = [p.get("slot", SLOT) for p in plan]
    need = [i for i, p in enumerate(plan) if "proof" not in p]
    got = _sign(eng, [(sk(plan[i]["g"]) if plan[i]["g"] < N_VAL else 1) + ("proof" in plan[i].get("bad", ())) for i in need],
                [C.signing_root(C.selection_data_root(slot[i], plan[i]["s"]), doms[32:64]) for i in need])
    proofs = [p.get("proof") for p in plan]
    for i, x in zip(need, got):
        proofs[i] = x

    def contrib_key(p):
        s = p["s"] % count
        return sum(sk(pv[s * sub + i]) for i, b in enumerate(p["bits"][:sub]) if b) + ("sig" in p.get("bad", ()))

    sigs = _sign(eng, [contrib_key(p) for p in plan], [C.signing_root(p["root"], doms[:32]) for p in plan])
    rows = [C.pack(p["bits"]) for p in plan]
    caps = [C.signing_root(C.contribution_and_proof_root(p["g"], slot[a], p["root"], p["s"], rows[a], sigs[a], proofs[a]), doms[64:96])
            for a, p in enumerate(plan)]
    outers = _sign(eng, [(sk(p["g"]) if p["g"] < N_VAL else 1) + ("outer" in p.get("bad", ())) for p in plan], caps)
    return [C.encode(p["g"], slot[a], p["root"], p["s"], p["bits"], sigs[a], proofs[a], outers[a]) for a, p in enumerate(plan)]


def _scc_expect(eng, plan, wires, pv, count, target, current_slot=SLOT, doms=DOMS):
    def ok(a, which):      # a given proof is never the aggregator's own signature
        p = plan[a]
        return which not in p.get("bad", ()) and "proof" not in p
    want = C.validate(wires, [int(x) for x in pv], N_VAL, lambda v: None, current_slot, doms, target=target, count=count,
                      verify=lambda a, pk, m, s, which: ok(a, ("proof", "outer")[which]), fast_verify=lambda a, keys, m, s: ok(a, "sig"),
                      secret_key=sk, closed_form=True)
    return M.sign_closed_form(want, lambda ks, ms: _sign(eng, ks, ms))


def _scc_dev(eng, wires, pv, count, slot, target):
    wire = np.frombuffer(b"".join(wires), np.uint8)
    r = eng.sync_contribution_and_proof_intake_dev(_t(wire), _t(_woff(wires)), _t(np.asarray(pv, np.uint32)), count, slot, DOMS, target)
    torch.cuda.synchronize()
    out = [x.cpu().numpy() for x in r]
    out[1], out[3] = out[1].view(np.uint32), out[3].view(np.uint32)
    return out


def _scc_run(eng, wires, pv, count, slot, target, want):
    w = C.expect_arrays(want, count=count, size=len(pv))
    host = eng.sync_contribution_and_proof_intake(b"".join(wires), _woff(wires), pv, count, slot, DOMS, target)
    _assert_equal(host, w, SCC_NAMES)
    _assert_equal(_scc_dev(eng, wires, pv, count, slot, target), w, SCC_NAMES)
    return host


def _aggregator_committee(eng, size, count, target, rng, per_subnet=4, slot=SLOT, doms=DOMS):
    """a committee whose subnets hold, at positions sub - 1, 0, 1, ..., up to per_subnet members whose own selection proof selects them
    at this modulus, and elsewhere members it does not select (modulus > 1) -> (pv, aggregators per subnet, non-aggregators per subnet)"""
    sub = size // count
    m = max(1, sub // target)
    cand = rng.permutation(N_VAL - 1)[:min(N_VAL - 1, max(2048, 6 * size))].tolist()
    sel = {}
    for s in range(count):
        pr = _proofs(eng, cand, [s] * len(cand), slot, doms)
        sel[s] = [v for v, p in zip(cand, pr) if C.is_aggregator(p, sub, target)]
    pv, used, aggs, non = [None] * size, set(), {}, {}
    for s in range(count):
        k = min(per_subnet, sub)
        aggs[s] = [v for v in sel[s] if v not in used][:k]
        assert len(aggs[s]) == k, (s, m, len(sel[s]))
        used.update(aggs[s])
        slots = [s * sub + sub - 1] + [s * sub + i for i in range(k - 1)]
        for p, v in zip(slots, aggs[s]):
            pv[p] = v
    selecting = set().union(*sel.values()) if m > 1 else set()
    rest = iter(v for v in cand if v not in used and v not in selecting)
    for p in range(size):
        if pv[p] is None:
            pv[p] = next(rest)
    for s in range(count):
        non[s] = [v for v in pv[s * sub:(s + 1) * sub] if v not in aggs[s]]
    return np.array(pv, np.uint32), aggs, non


@pytest.mark.parametrize("size,count,target", SHAPES, ids=["%dx%d" % s[:2] for s in SHAPES])
def test_contribution_shapes(env, size, count, target):
    """per subnet: the last position's bit alone (accepted), a padding bit (1), a check-8 subset and a superset that differ from the
    accepted row only in its last partial word (8, then accepted), a second root of a seen aggregator (9), a member whose proof does not
    select (5); the aggregates through b2_sync_aggregate_verify"""
    eng, pks = env
    t0 = time.perf_counter()
    rng = np.random.default_rng(size * 7 + count)
    sub, m = size // count, max(1, (size // count) // target)
    sb, sw = (sub + 7) // 8, ((sub + 7) // 8 + 3) // 4
    pv, aggs, non = _aggregator_committee(eng, size, count, target, rng)
    ra, rb = bytes([0x30 + count]) * 32, bytes([0x40 + count]) * 32
    bits = lambda *ix: [i in ix for i in range(8 * sb)]      # noqa: E731
    plan = []
    for s in range(count):
        a = aggs[s]
        plan.append(dict(g=a[0], s=s, root=ra, bits=bits(sub - 1)))                   # 0: bit sub - 1 alone
        if sub & 7:
            plan.append(dict(g=a[-1], s=s, root=ra, bits=bits(0, sub)))               # 1: the first padding bit
            plan.append(dict(g=a[-1], s=s, root=ra, bits=bits(8 * sb - 1)))           # 1: the last padding bit
        plan.append(dict(g=a[0], s=s, root=rb, bits=bits(0)))                         # 9: a second root
        if len(a) >= 3:
            j = (32 * (sw - 1) + sub - 1) // 2                                          # a bit of the last word, not 0 or sub - 1
            assert 32 * (sw - 1) <= j < sub and j not in (0, sub - 1)
            plan.append(dict(g=a[1], s=s, root=rb, bits=bits(0, sub - 1)))            # 0
            plan.append(dict(g=a[2], s=s, root=rb, bits=bits(sub - 1)))               # 8: a subset
            plan.append(dict(g=a[2], s=s, root=rb, bits=bits(0, sub - 1, j)))         # 0: a superset only in the last word
        if m > 1:
            plan.append(dict(g=non[s][0], s=s, root=ra, bits=bits(0)))                # 5
    wires = _scc_wires(eng, plan, pv, sub, count)
    want = _scc_expect(eng, plan, wires, pv, count, target)
    st = set(want.status)
    assert 0 in st and 9 in st
    assert (1 in st) == bool(sub & 7) and (8 in st) == (sub >= 3) and (5 in st) == (m > 1)
    host = _scc_run(eng, wires, pv, count, SLOT, target, want)
    _verify_aggregates(eng, pks, pv, want.roots, host.agg_bits, host.agg_sigs)
    _timed("contributions %dx%d, sub %d, modulus %d, %d items" % (size, count, sub, m, len(wires)), t0)


def test_shape_list_reaches_every_class():
    subs = {s // c for s, c, _ in SHAPES}
    assert subs == {1, 9, 40, 125, 510, 260, 768, 1024, 256, 128}
    assert {max(1, (s // c) // t) for s, c, t in SHAPES} == {1, 3, 7, 8, 64, 341}
    assert any(t > s // c for s, c, t in SHAPES)
    chunks = {((s // c + 7) // 8 + 31) // 32 for s, c, _ in SHAPES}
    assert chunks == {1, 2, 3, 4}


# ------------------------------------------------------------------------------------------------------------ colliding roots

@pytest.mark.parametrize("n,k", [(1, 1), (2, 2), (3, 3), (64, 33), (65, 33), (64, 64), (4096, 257)])
def test_message_colliding_roots(env, n, k):
    """k distinct roots on slot tab - 1 (every probe past the first wraps to slot 0 and on), byte-equal copies behind the chain, the rest
    of the n items rejected; (64, 64): every root of the call on one slot"""
    eng, pks = env
    t0 = time.perf_counter()
    tab = K.table_size(n)
    roots = K.colliding(k, tab - 1, tab, tag=n)
    size, count = 1024, 4
    pv = np.arange(1, size + 1, dtype=np.uint32)
    items, subnets = [], []
    for a in range(n):
        p = a % size
        if a < k:
            items.append((SLOT, roots[a], int(pv[p]), None))                                   # a new root
        elif a < size:
            items.append((SLOT, roots[(a * 7) % k], int(pv[p]), None))                          # a copy behind the chain
        else:
            items.append((SLOT, roots[a % k], int(pv[p]), None))                               # 5: seen
        subnets.append(p // (size // count))
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, subnets, pv, count, SLOT)
    assert want.roots == roots and want.status.count(0) == min(n, size)
    assert all(K.home_slot(r, tab) == tab - 1 for r in want.roots)      # k >= 2: the second root's probe wraps to slot 0
    _msg_run(eng, wires, subnets, pv, count, SLOT, want)
    _timed("messages, %d roots on one slot of %d, n %d" % (k, tab, n), t0)


@pytest.mark.parametrize("n", [3, 64, 65, 4096])
def test_contribution_colliding_roots(env, n):
    """R and R' distinct on one home slot (the chain wraps): A accepted on R with bits S; B on R' with bits within S from another
    aggregator is accepted (not covered: another root); C on a byte-equal copy of R with bits within S is 8; roots first entered by items
    that fail 10, 11 or 12 and later accepted from items with the same bytes; the rest of the n items of another slot (2)"""
    eng, pks = env
    t0 = time.perf_counter()
    size, count, target = 64, 4, 16      # sub 16, modulus 1: every proof selects
    sub = size // count
    pv = np.arange(100, 100 + size, dtype=np.uint32)
    tab = K.table_size(n)
    kk = min(33, max(3, n // 2))
    rs = K.colliding(kk, tab - 1, tab, tag=n)
    R0, R1 = rs[0], rs[1]
    bits = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    g = lambda s, i: int(pv[s * sub + i])                 # noqa: E731
    plan = [dict(g=g(0, 0), s=0, root=R0, bits=bits(0, 1, 2, 3)),        # A: 0
            dict(g=g(0, 1), s=0, root=R1, bits=bits(1, 2)),              # B: 0 (R1 collides with R0 but is another root)
            dict(g=g(0, 2), s=0, root=bytes(R0), bits=bits(2, 3))]       # C: 8
    if n > 3:
        for j, bad in enumerate(("proof", "outer", "sig")):
            r = rs[2 + j]
            plan.append(dict(g=g(1 + j, 0), s=1 + j, root=r, bits=bits(0, 5), bad={bad}))       # 10, 11, 12: the root enters the table
            plan.append(dict(g=g(1 + j, 1), s=1 + j, root=bytes(r), bits=bits(1, 5)))            # 0 from the same bytes
        for j in range(5, kk):                                                                     # the rest of the chain
            s, i = j % count, 2 + j // count
            plan.append(dict(g=g(s, i), s=s, root=rs[j], bits=bits(i)))
    while len(plan) < n:
        plan.append(dict(g=g(0, 5), s=0, root=R0, bits=bits(5), slot=SLOT + 1))               # 2
    wires = _scc_wires(eng, plan, pv, sub, count)
    want = _scc_expect(eng, plan, wires, pv, count, target)
    assert want.status[:3] == [0, 0, 8]
    if n > 3:
        assert want.status[3:9] == [10, 0, 11, 0, 12, 0] and len(want.roots) == kk
    host = _scc_run(eng, wires, pv, count, SLOT, target, want)
    _verify_aggregates(eng, pks, pv, want.roots, host.agg_bits, host.agg_sigs)
    _timed("contributions, %d roots on one slot of %d, n %d" % (len(want.roots), tab, n), t0)


# ------------------------------------------------------------------------------------------------------------ past one CTA of roots

def test_message_roots_past_one_cta(env):
    """1 100 rejected items (subnet >= count) first, then 1 024 positions signing 1 024 distinct roots, then duplicates naming early roots:
    every root leader sits at list index >= 1 024, reaching k_scm_number's third chunk"""
    eng, pks = env
    t0 = time.perf_counter()
    size, count = 1024, 4
    pv = np.arange(2000, 2000 + size, dtype=np.uint32)
    roots = [K.root_at(j % 4096, 4096, tag=j) for j in range(size)]
    items, subnets = [], []
    for a in range(1100):
        items.append((SLOT, roots[a % size], int(pv[a % size]), None))
        subnets.append(count)
    for p in range(size):
        items.append((SLOT, roots[p], int(pv[p]), None))
        subnets.append(p // 256)
    for p in range(0, 400, 2):
        items.append((SLOT, roots[p + 1], int(pv[p]), None))
        subnets.append(p // 256)
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, subnets, pv, count, SLOT)
    leaders = [want.root_id.index(r) for r in range(len(want.roots))]
    assert len(want.roots) == 1024 and min(leaders) >= 1024 and max(leaders) >= 2048
    assert set(want.status) == {0, 4, 5}
    host = _msg_run(eng, wires, subnets, pv, count, SLOT, want)
    _verify_aggregates(eng, pks, pv, want.roots[:64], host.agg_bits[:64], host.agg_sigs[:64])
    _timed("messages, 1 024 roots after 1 100 rejected items", t0)


def test_contribution_roots_past_one_cta(env):
    """1 100 items of another slot first, then 1 000 aggregators (target >= sub: every proof selects) on 1 000 roots across 4 subnets, and
    24 later aggregators tying on early (root, subnet)s with disjoint rows of equal popcount more than 128 list positions later (another
    CTA of k_scc_best): the earlier item stays best"""
    eng, pks = env
    t0 = time.perf_counter()
    size, count = 1024, 4
    sub = size // count
    pv = np.arange(1000, 1000 + size, dtype=np.uint32)
    roots = [K.root_at((j * 5) % 4096, 4096, tag=j + 7) for j in range(1000)]
    bits = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    plan = [dict(g=int(pv[a % size]), s=(a % size) // sub, root=roots[a % 1000], bits=bits(0), slot=SLOT + 2) for a in range(1100)]
    first = {}
    for j in range(1000):
        p = (j % 4) * sub + j // 4                                      # subnet j % 4, position j // 4 of it
        first[j] = len(plan)
        plan.append(dict(g=int(pv[p]), s=j % 4, root=roots[j], bits=bits(j // 4)))
    ties = []
    for t in range(24):
        j = 4 * t + (t % 4)                                             # an early root of subnet j % 4
        p = (j % 4) * sub + 250 + t // 4
        ties.append((j, len(plan)))
        plan.append(dict(g=int(pv[p]), s=j % 4, root=roots[j], bits=bits(250 + t // 4)))
    wires = _scc_wires(eng, plan, pv, sub, count)
    want = _scc_expect(eng, plan, wires, pv, count, sub)
    leaders = [want.root_id.index(r) for r in range(len(want.roots))]
    assert len(want.roots) == 1000 and min(leaders) >= 1024 and max(leaders) >= 2048
    assert want.status.count(0) == 1024
    for j, a in ties:
        r = want.roots.index(roots[j])
        assert want.best[r][j % 4] == first[j] and a - first[j] > 128
    _scc_run(eng, wires, pv, count, SLOT, sub, want)
    _timed("contributions, 1 000 roots after 1 100 rejected items", t0)


# ------------------------------------------------------------------------------------------------------------ u64 fields

def test_message_u64_fields(env):
    eng, pks = env
    size, count = 32, 4
    pv = np.arange(40, 40 + size, dtype=np.uint32)
    ra = bytes([0x5A]) * 32
    v0 = int(pv[3])
    items = [(SLOT, ra, (1 << 32) + v0, sk(v0)), (SLOT, ra, (1 << 63) + v0, sk(v0)), (SLOT, ra, U64, sk(v0)),     # 3
             (SLOT + (1 << 32), ra, v0, None),                                                                     # 2
             (SLOT, ra, v0, None)]                                                                                 # 0
    subnets = [0] * len(items)
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, subnets, pv, count, SLOT)
    assert want.status == [3, 3, 3, 2, 0]
    _msg_run(eng, wires, subnets, pv, count, SLOT, want)
    items = [(U64, ra, v0, None), (U64, ra, int(pv[9]), None), (U64 - (1 << 32), ra, v0, None)]
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, [0, 1, 0], pv, count, U64)
    assert want.status == [0, 0, 2]
    _msg_run(eng, wires, [0, 1, 0], pv, count, U64, want)


def test_contribution_u64_fields(env):
    """every proof selects (target >= sub): aggregator_index 2^32 + v is 6, subcommittee_index 2^32 + s and 2^64 - 1 are 3, a slot with a
    high word is 2; current_slot 2^64 - 1 is accepted"""
    eng, pks = env
    size, count = 32, 4
    sub = size // count
    pv = np.arange(40, 40 + size, dtype=np.uint32)
    ra = bytes([0x6B]) * 32
    v1 = int(pv[sub + 2])
    bits = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    plan = [dict(g=(1 << 32) + v1, s=1, root=ra, bits=bits(2)),
            dict(g=v1, s=(1 << 32) + 1, root=ra, bits=bits(2)),
            dict(g=v1, s=U64, root=ra, bits=bits(2)),
            dict(g=v1, s=1, root=ra, bits=bits(2), slot=SLOT + (1 << 32)),
            dict(g=v1, s=1, root=ra, bits=bits(2))]
    wires = _scc_wires(eng, plan, pv, sub, count)
    want = _scc_expect(eng, plan, wires, pv, count, sub)
    assert want.status == [6, 3, 3, 2, 0]
    _scc_run(eng, wires, pv, count, SLOT, sub, want)
    plan = [dict(g=v1, s=1, root=ra, bits=bits(2, 3), slot=U64), dict(g=int(pv[0]), s=0, root=ra, bits=bits(0), slot=U64)]
    wires = _scc_wires(eng, plan, pv, sub, count)
    want = _scc_expect(eng, plan, wires, pv, count, sub, current_slot=U64)
    assert want.status == [0, 0]
    _scc_run(eng, wires, pv, count, U64, sub, want)


# ------------------------------------------------------------------------------------------------------------ exceptional sums

def _eth_verify_aggregates(pks, pv, want, dom):
    """the aggregates' verdicts from the upstream rule (eth_fast_aggregate_verify over the set positions' keys)"""
    out = []
    for root, a in zip(want.roots, want.aggregates):
        keys = [pks[int(pv[p])].tobytes() for p, b in enumerate(a.sync_committee_bits) if b]
        out.append(SO.eth_fast_aggregate_verify(keys, M.signing_root(root, dom), a.sync_committee_signature))
    return out


@pytest.mark.parametrize("case", ["p_and_p_plus_32", "whole_subnet", "whole_committee", "negated_key"])
def test_message_exceptional_sums(env, case):
    """P + P in one lane of the segment sums (one validator at positions p and p + 32, or on a whole subnet or committee) and P + (-P) (the
    validator holding r - sk(0) beside validator 0): statuses and bytes against the oracle, the aggregates' verdicts against
    eth_fast_aggregate_verify, and through b2_sync_aggregate_verify where they are not the point at infinity"""
    eng, pks = env
    size, count = (512, 1) if case == "whole_committee" else (128, 2)
    sub = size // count
    pv = np.arange(300, 300 + size, dtype=np.uint32)
    if case == "p_and_p_plus_32":
        pv[5 + 32] = pv[5]
        pv[sub + 20 + 32] = pv[sub + 20]
    elif case == "whole_subnet":
        pv[sub:2 * sub] = 77
    elif case == "whole_committee":
        pv[:] = 78
    else:
        pv[3], pv[3 + 32] = 0, N_VAL - 1
        pv[sub + 3], pv[sub + 9] = 0, N_VAL - 1
    ra = bytes([0x7C]) * 32
    pairs = sorted({(int(pv[p]), p // sub) for p in range(size)}, key=lambda x: (x[1], x[0]))
    items = [(SLOT, ra, v, None) for v, s in pairs]
    subnets = [s for v, s in pairs]
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, subnets, pv, count, SLOT)
    assert set(want.status) == {0}
    host = _msg_run(eng, wires, subnets, pv, count, SLOT, want)
    assert _eth_verify_aggregates(pks, pv, want, DOM) == [True]
    if case == "negated_key":      # P and -P in one lane of subnet 0's sum (positions 3 and 35), and in the root's
        assert all(want.contributions[(0, 0)].aggregation_bits[i] for i in (3, 35))
    elif case == "whole_committee":
        assert want.aggregates[0].sync_committee_signature == _sign(eng, [512 * sk(78)], [M.signing_root(ra, DOM)])[0]
    _verify_aggregates(eng, pks, pv, want.roots, host.agg_bits, host.agg_sigs)


def test_message_sum_at_infinity(env):
    """a subnet whose only signers are validator 0 and the holder of -sk(0), in one lane (positions 3 and 35): that contribution's sum
    and the root's aggregate are the point at infinity (0xc0 || 0^95), as bls.Aggregate gives"""
    eng, pks = env
    size, count = 64, 1
    pv = np.arange(500, 500 + size, dtype=np.uint32)
    pv[3], pv[35] = 0, N_VAL - 1
    ra = bytes([0x7D]) * 32
    items = [(SLOT, ra, 0, None), (SLOT, ra, N_VAL - 1, None)]
    wires = _msg_wires(eng, items)
    want = _msg_expect(eng, items, wires, [0, 0], pv, count, SLOT)
    assert want.status == [0, 0] and want.aggregates[0].sync_committee_signature == INF
    assert want.contributions[(0, 0)].signature == INF
    _msg_run(eng, wires, [0, 0], pv, count, SLOT, want)
    assert _eth_verify_aggregates(pks, pv, want, DOM) == [False]      # the keys sum to infinity too: eth_fast_aggregate_verify refuses


def test_contribution_exceptional_sums(env):
    """real signatures through the oracle's own verification: one validator at positions p and p + 32 of a subnet in one contribution;
    a subnet of one validator; a contribution whose set keys cancel (validator 0 and the holder of -sk(0)); two contributions on one
    root whose sum is the point at infinity"""
    eng, pks = env
    size, count = 256, 4
    sub = size // count
    pv = np.arange(600, 600 + size, dtype=np.uint32)
    pv[5 + 32] = pv[5]                       # subnet 0: one validator in one lane twice
    pv[sub:2 * sub] = 91                     # subnet 1: one validator
    pv[2 * sub + 3], pv[2 * sub + 4] = 0, N_VAL - 1      # subnet 2: keys that cancel, and -sk(0) again at position 7
    pv[2 * sub + 7] = N_VAL - 1
    pv[3 * sub] = 0                                      # subnet 3: sk(0)
    ra, rb = bytes([0x31]) * 32, bytes([0x32]) * 32
    bits = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    plan = [dict(g=int(pv[5]), s=0, root=ra, bits=bits(5, 37, 9)),
            dict(g=91, s=1, root=ra, bits=[True] * sub),
            dict(g=0, s=2, root=ra, bits=bits(3, 4)),                   # keys cancel: the signature is infinity
            dict(g=N_VAL - 1, s=2, root=rb, bits=bits(7)),             # -sk(0) alone on root B, subnet 2
            dict(g=0, s=3, root=rb, bits=bits(0))]                     # sk(0) alone on root B, subnet 3: root B sums to infinity
    wires = _scc_wires(eng, plan, pv, sub, count)
    pk = lambda v: pks[v].tobytes()      # noqa: E731
    want = C.validate(wires, [int(x) for x in pv], N_VAL, pk, SLOT, DOMS, target=sub, count=count)
    assert want.status == [0, 0, 12, 0, 0]      # the cancelling contribution fails FastAggregateVerify (its keys sum to infinity)
    assert want.aggregates[want.roots.index(rb)].sync_committee_signature == INF
    got = _scc_run(eng, wires, pv, count, SLOT, sub, want)
    verdict = []
    for root, a in zip(want.roots, want.aggregates):
        keys = [pk(int(pv[p])) for p, b in enumerate(a.sync_committee_bits) if b]
        verdict.append(SO.eth_fast_aggregate_verify(keys, M.signing_root(root, DOMS[:32]), a.sync_committee_signature))
    assert verdict == [True, False]      # root B: keys and signature at infinity
    _verify_aggregates(eng, pks, pv, want.roots[:1], got.agg_bits[:1], got.agg_sigs[:1])


# ------------------------------------------------------------------------------------------------------------ rows past n_roots

def _sentinel(shape, dtype):
    return torch.full(shape if isinstance(shape, tuple) else (shape,), SENTINEL, dtype=dtype, device=torch.device("cuda", 0))


def test_rows_past_n_roots(env):
    """the device forms with trim=False into sentinel-filled tensors, and the raw host calls into sentinel arrays: every row past n_roots
    is written as include/b200pos.h states (zero; best 0xFFFFFFFF)"""
    eng, pks = env
    size, count, sub = 64, 4, 16
    pv = np.arange(700, 700 + size, dtype=np.uint32)
    ra, rb = bytes([0x41]) * 32, bytes([0x42]) * 32
    items = [(SLOT, ra, int(pv[p]), None) for p in range(0, size, 3)] + [(SLOT, rb, int(pv[1]), None), (SLOT + 1, ra, int(pv[2]), None)]
    subnets = [p // sub for p in range(0, size, 3)] + [0, 0]
    wires = _msg_wires(eng, items)
    n = len(wires)
    want = _msg_arrays(_msg_expect(eng, items, wires, subnets, pv, count, SLOT), size, count)
    k = len(want[2])
    u8, i32 = torch.uint8, torch.int32
    out = (SyncMessagesResult(_sentinel(n, i32), _sentinel(n, i32), _sentinel((n, 32), u8), _sentinel((n, count, 2), u8), _sentinel((n, count, 96), u8),
                 _sentinel((n, count), u8), _sentinel((n, 8), u8), _sentinel((n, 96), u8)), _sentinel(1, i32))
    wire = np.frombuffer(b"".join(wires), np.uint8)
    res, nr = eng.sync_committee_messages_dev(_t(wire), _t(_woff(wires)), _t(np.asarray(subnets, np.uint32)), _t(pv), count, SLOT, DOM,
                                              out=out, trim=False)
    torch.cuda.synchronize()
    assert int(nr.item()) == k == 2
    got = [x.cpu().numpy() for x in res]
    got[1] = got[1].view(np.uint32)
    for name, g, w in zip(MSG_NAMES, got, want):
        if name in ("status", "root_id"):
            assert np.array_equal(g.astype(w.dtype), w), name
        else:
            assert np.array_equal(g[:k], w), name
            assert (g[k:] == 0).all(), name
    # the raw host call
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)      # noqa: E731
    outs = [np.full(n, SENTINEL, np.int32), np.full(n, SENTINEL, np.uint32), np.full((n, 32), SENTINEL, np.uint8), np.full(1, SENTINEL, np.uint32),
            np.full((n, count, 2), SENTINEL, np.uint8), np.full((n, count, 96), SENTINEL, np.uint8), np.full((n, count), SENTINEL, np.uint8),
            np.full((n, 8), SENTINEL, np.uint8), np.full((n, 96), SENTINEL, np.uint8)]
    wo, sn, pvv = _woff(wires), np.asarray(subnets, np.uint32), np.asarray(pv, np.uint32)
    dom = np.frombuffer(DOM, np.uint8).copy()
    assert eng.lib.b2_sync_committee_messages(eng.h, p(wire), len(wire), p(wo), n, p(sn), p(pvv), size, count, SLOT, p(dom),
                                              *[p(o) for o in outs]) == 0
    assert outs[3][0] == k
    for name, g, w in zip(MSG_NAMES, [outs[0], outs[1], outs[2]] + outs[4:], want):
        assert np.array_equal(g[:k] if name not in ("status", "root_id") else g, w), name
        if name not in ("status", "root_id"):
            assert (g[k:] == 0).all(), name
    # contributions
    bits = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    plan = [dict(g=int(pv[0]), s=0, root=ra, bits=bits(0, 3)), dict(g=int(pv[17]), s=1, root=rb, bits=bits(1)),
            dict(g=int(pv[18]), s=1, root=rb, bits=bits(1), slot=SLOT + 1), dict(g=int(pv[33]), s=2, root=ra, bits=bits(1), bad={"sig"})]
    wires = _scc_wires(eng, plan, pv, sub, count)
    n = len(wires)
    want = C.expect_arrays(_scc_expect(eng, plan, wires, pv, count, sub), count=count, size=size)
    k = len(want[2])
    out = (SyncContributionsResult(_sentinel(n, i32), _sentinel(n, i32), _sentinel((n, 32), u8), _sentinel((n, count), i32), _sentinel((n, 8), u8),
                 _sentinel((n, 96), u8)), _sentinel(1, i32))
    wire = np.frombuffer(b"".join(wires), np.uint8)
    res, nr = eng.sync_contribution_and_proof_intake_dev(_t(wire), _t(_woff(wires)), _t(pv), count, SLOT, DOMS, sub, out=out, trim=False)
    torch.cuda.synchronize()
    assert int(nr.item()) == k == 2
    got = [x.cpu().numpy() for x in res]
    got[1], got[3] = got[1].view(np.uint32), got[3].view(np.uint32)
    outs = [np.full(n, SENTINEL, np.int32), np.full(n, SENTINEL, np.uint32), np.full((n, 32), SENTINEL, np.uint8), np.full(1, SENTINEL, np.uint32),
            np.full((n, count), SENTINEL, np.uint32), np.full((n, 8), SENTINEL, np.uint8), np.full((n, 96), SENTINEL, np.uint8)]
    dom = np.frombuffer(DOMS, np.uint8).copy()
    assert eng.lib.b2_sync_contribution_and_proof_intake(eng.h, p(wire), len(wire), p(_woff(wires)), n, p(pvv), size, count, SLOT, p(dom), sub,
                                                         *[p(o) for o in outs]) == 0
    assert outs[3][0] == k
    for form in (got, [outs[0], outs[1], outs[2]] + outs[4:]):
        for name, g, w in zip(SCC_NAMES, form, want):
            if name in ("status", "root_id"):
                assert np.array_equal(g.astype(w.dtype), w), name
                continue
            assert np.array_equal(g[:k], w), name
            assert (g[k:] == (0xFFFFFFFF if name == "best" else 0)).all(), name


# ------------------------------------------------------------------------------------------------------------ interleaving

def _interleaved_calls(eng):
    """the inputs of: messages at 1 024 positions / n = 3 000; contributions at 32 / n = 5; b2_aggregate_verify; contributions at 1 024
    / n = 4 096; messages at n = 3"""
    rng = np.random.default_rng(99)
    pv1k = np.arange(1500, 2524, dtype=np.uint32)
    ra, rb = bytes([0x51]) * 32, bytes([0x52]) * 32
    items, subnets = [], []
    for a in range(3000):
        p = int(rng.integers(0, 1024))
        items.append((SLOT, (ra, rb)[a % 2], int(pv1k[p]), None if rng.random() > 0.1 else 5))
        subnets.append(p // 256)
    m1 = (_msg_wires(eng, items), subnets, pv1k)
    pv32 = np.arange(50, 82, dtype=np.uint32)
    b8 = lambda *ix: [i in ix for i in range(8)]      # noqa: E731
    plan = [dict(g=int(pv32[s * 8 + 1]), s=s, root=ra, bits=b8(1, s)) for s in range(4)] + [dict(g=int(pv32[2]), s=0, root=rb, bits=b8(2))]
    c1 = (_scc_wires(eng, plan, pv32, 8, 4), pv32, 8)
    plan = []
    for a in range(4096):
        p = int(rng.integers(0, 1024))
        plan.append(dict(g=int(pv1k[p]), s=p // 256, root=(ra, rb)[a % 2], bits=[bool(x) for x in rng.random(256) < 0.3]))
    c2 = (_scc_wires(eng, plan, pv1k, 256, 4), pv1k, 256)
    m2 = (_msg_wires(eng, [(SLOT, ra, int(pv32[0]), None), (SLOT, rb, int(pv32[9]), None), (SLOT, ra, int(pv32[0]), None)]), [0, 1, 0], pv32)
    msgs = np.frombuffer(M.signing_root(ra, DOM), np.uint8).reshape(1, 32)
    av = ([3, 4, 5], [0, 1, 2, 3], np.repeat(msgs, 3, 0), np.stack([np.frombuffer(s, np.uint8) for s in
                                                                    _sign(eng, [sk(3), sk(4), sk(5) + 1], [msgs[0].tobytes()] * 3)]))
    return m1, c1, av, c2, m2


def _fresh_sequence(pks, calls, rlc):
    out = []
    for j in range(5):
        e = _fresh(pks)
        try:
            if rlc:
                e.set_verify_mode(True, bytes(range(32)))
            out.append(_run_sequence_one(e, calls, j))
        finally:
            e.close()
    return out


def _run_sequence_one(eng, calls, j):
    m1, c1, av, c2, m2 = calls
    if j == 0:
        return _msg_dev(eng, m1[0], m1[1], m1[2], 4, SLOT)
    if j == 1:
        return _scc_dev(eng, c1[0], c1[1], 4, SLOT, c1[2])
    if j == 2:
        return [eng.aggregate_verify(*av)]
    if j == 3:
        return _scc_dev(eng, c2[0], c2[1], 4, SLOT, c2[2])
    return list(eng.sync_committee_messages(b"".join(m2[0]), _woff(m2[0]), m2[1], m2[2], 4, SLOT, DOM))


def test_interleaved_call_families(env):
    """messages, contributions and b2_aggregate_verify share the AggregateVerify buffers and pipeline slot 0's verify buffers, each family
    growing its scratch as it goes: one engine runs the sequence twice (the second time in the RLC verify mode), and every call's outputs
    equal a fresh engine's"""
    eng, pks = env
    t0 = time.perf_counter()
    calls = _interleaved_calls(eng)
    eng.set_verify_mode(False)
    for rlc in (False, True):
        if rlc:
            eng.set_verify_mode(True, bytes(range(32)))
        try:
            got = [_run_sequence_one(eng, calls, j) for j in range(5)]
        finally:
            eng.set_verify_mode(False)
        want = _fresh_sequence(pks, calls, rlc)
        for j, (g, w) in enumerate(zip(got, want)):
            assert len(g) == len(w), j
            for x, y in zip(g, w):
                assert np.array_equal(np.asarray(x), np.asarray(y)), (rlc, j)
    st = np.asarray(got[0][0])
    assert {0, 5, 6} <= set(st.tolist()) and got[2][0].tolist() == [1, 1, 0]
    assert set(np.asarray(got[3][0]).tolist()) >= {0, 9}
    _timed("interleaved sequence, twice, against fresh engines", t0)


# ------------------------------------------------------------------------------------------------------------ Spec facades, mainnet preset

def test_spec_facades_mainnet_preset():
    """Spec.validate_sync_committee_messages and Spec.validate_sync_contribution_and_proofs on the mainnet preset (512 positions, 4 subnets of
    128, target 16: aggregator modulus 8): a committee with repeated keys, a subnet id of 2^32 + 1 (status 4, not subnet 1), and the
    contributions at the period boundary, where the next committee is the one checked"""
    import dataclasses
    from pos_evolution_b200 import spec as PS
    P = PS.MAINNET
    t0 = time.perf_counter()
    eng = Engine(0)
    try:
        pks = eng.sk_to_pk([sk(v) for v in range(N_VAL)])
        rng = np.random.default_rng(512)
        cur = _committee(512, rng)
        cur[1] = cur[2] = cur[3]
        cur[200] = cur[300] = cur[100]
        state = PS.BeaconState(slot=5000, fork=PS.Fork(bytes([1, 0, 0, 0]), bytes([2, 0, 0, 0]), 0), genesis_validators_root=bytes(range(32)),
                               validators=[PS.Validator(pks[v].tobytes(), 32 * 10**9, False, 0, U64) for v in range(N_VAL)],
                               balances=[32 * 10**9] * N_VAL, randao_mixes=[bytes(32)] * P.EPOCHS_PER_HISTORICAL_VECTOR,
                               block_roots=[bytes(32)] * P.SLOTS_PER_HISTORICAL_ROOT, previous_epoch_participation=[0] * N_VAL,
                               current_epoch_participation=[0] * N_VAL)
        state.current_sync_committee = PS.SyncCommittee([pks[v].tobytes() for v in cur], bytes(48))
        pspec = PS.Spec(P, engine=eng)
        assert P.SYNC_COMMITTEE_SIZE == 512 and P.SYNC_COMMITTEE_SUBNET_COUNT == 4 and P.TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE == 16
        boundary = P.SLOTS_PER_EPOCH * P.EPOCHS_PER_SYNC_COMMITTEE_PERIOD - 1
        ep = pspec.compute_epoch_at_slot(boundary)
        doms_b = b"".join(pspec.get_domain(state, d, ep) for d in (PS.DOMAIN_SYNC_COMMITTEE, PS.DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF,
                                                                     PS.DOMAIN_CONTRIBUTION_AND_PROOF))
        nxt, aggs, non = _aggregator_committee(eng, 512, 4, 16, rng, slot=boundary, doms=doms_b)
        nxt[7] = nxt[8]
        state.next_sync_committee = PS.SyncCommittee([pks[v].tobytes() for v in nxt], bytes(48))
        # messages at slot 5000: the current committee
        dom = pspec.get_domain(state, PS.DOMAIN_SYNC_COMMITTEE, pspec.compute_epoch_at_slot(state.slot))
        ra, rb = bytes([0x61]) * 32, bytes([0x62]) * 32
        pairs = sorted({(int(cur[p]), p // 128) for p in range(512)}, key=lambda x: (x[1], x[0]))
        items = [(state.slot, (ra, rb)[j % 3 == 0], v, None if j % 17 else sk(v) + 1) for j, (v, s) in enumerate(pairs)]
        subnets = [s for v, s in pairs]
        items.append((state.slot, ra, int(cur[128 + 9]), None))
        subnets.append((1 << 32) + 1)                                         # cur[137] is on subnet 1: the id's high word counts
        wires = _msg_wires(eng, items, dom)
        want = _msg_expect(eng, items, wires, subnets, cur, 4, state.slot, dom)
        assert want.status[-1] == 4 and {0, 6} <= set(want.status) and len(want.roots) == 2
        msgs = [(s, PS.SyncCommitteeMessage(state.slot, w[8:40], int.from_bytes(w[40:48], "little"), w[48:144])) for w, s in zip(wires, subnets)]
        status, contributions, aggregates = pspec.validate_sync_committee_messages(state, msgs)
        assert status == want.status
        wc = [want.contributions[k] for k in sorted(want.contributions)]
        assert [(c.beacon_block_root, c.subcommittee_index, c.aggregation_bits, c.signature) for c in contributions] == \
            [(c.beacon_block_root, c.subcommittee_index, c.aggregation_bits, c.signature) for c in wc]
        assert list(aggregates) == want.roots
        for k, root in enumerate(want.roots):
            assert aggregates[root].sync_committee_bits == want.aggregates[k].sync_committee_bits
            assert aggregates[root].sync_committee_signature == want.aggregates[k].sync_committee_signature
        # contributions at the period boundary: the next committee
        b = dataclasses.replace(state, slot=boundary)
        outsider = next(int(v) for v in cur[128:256] if int(v) not in set(int(x) for x in nxt[128:256]))
        bits = lambda *ix: [i in ix for i in range(128)]      # noqa: E731
        plan = []
        for s in range(4):
            a = aggs[s]
            plan += [dict(g=a[0], s=s, root=ra, bits=bits(0, 5, 127)), dict(g=a[1], s=s, root=ra, bits=bits(5, 127)),
                     dict(g=a[0], s=s, root=rb, bits=bits(9)), dict(g=a[2], s=s, root=rb, bits=bits(127)), dict(g=non[s][0], s=s, root=ra, bits=bits(1))]
        plan.append(dict(g=outsider, s=1, root=ra, bits=bits(3), proof=_aggregator_proof(eng, outsider, 1, boundary, doms_b)))
        wires = _scc_wires(eng, [dict(p, slot=boundary) for p in plan], nxt, 128, 4, doms_b)
        want = _scc_expect(eng, plan, wires, nxt, 4, 16, boundary, doms_b)
        assert want.status == [0, 8, 9, 0, 5] * 4 + [7]
        items = []
        for w in wires:
            g, slot, root, s, row, sig, proof, outer = C.decode(w, 16)
            items.append(PS.SignedContributionAndProof(PS.ContributionAndProof(g, PS.SyncCommitteeContribution(slot, root, s, C._bits(row, 128), sig),
                                                                               proof), outer))
        status, aggregates = pspec.validate_sync_contribution_and_proofs(b, items)
        assert status == want.status and list(aggregates) == want.roots
        for k, root in enumerate(want.roots):
            assert aggregates[root].sync_committee_bits == want.aggregates[k].sync_committee_bits
            assert aggregates[root].sync_committee_signature == want.aggregates[k].sync_committee_signature
    finally:
        eng.close()
    _timed("Spec facades on the mainnet preset", t0)


def _aggregator_proof(eng, v, s, slot, doms):
    """a selection proof that selects at modulus 8 but is not v's own signature (its hash decides check 5; check 7 comes first)"""
    msg = C.signing_root(C.selection_data_root(slot, s), doms[32:64])
    for k in range(1, 400):
        p = _sign(eng, [sk(v) + k], [msg])[0]
        if C.is_aggregator(p, 128, 16):
            return p
    raise AssertionError("no selecting proof")
