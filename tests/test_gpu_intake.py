"""GPU parity of the attestation intake (Engine.attestation_intake / attestation_intake_dev, EpochProcessor.intake_dev): every status
0-13 and every output array against tests/intake_oracle.py, the max_votes overflow, the vote form fed by the intake end to end against
the BLS and fork-choice oracle and against the same epoch fed oracle-built votes, the tree's slot column after a prune and an add, the
host form's error contract, the device guards, and a full-size epoch of 2^20 attestations against the numpy oracle."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch

import intake_oracle as IO
import scenarios
from oracle import bls_sig as B
from oracle import fast
from oracle.ssz import compute_domain

pytestmark = pytest.mark.gpu

SPE, CPS, CSIZE, EPOCH = 8, 2, 7, 3
N_C = SPE * CPS
DOMAIN = compute_domain(bytes.fromhex("01000000"), bytes(4), bytes(32))
SENTINEL = 0xA5
FIELDS = ("status", "vote", "vote_off", "sigs", "data128", "msgs", "source_epoch", "target_epoch", "block_idx")


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _tree(seed=1, n_blocks=40, first_slot=EPOCH * SPE - 6):
    """a fork tree whose slots increase with the id, so along every chain"""
    rng = np.random.default_rng(seed)
    parent = np.array([0] + [max(0, b - 1 - int(rng.integers(0, 3))) for b in range(1, n_blocks)], dtype=np.uint32)
    slot = (first_slot + np.arange(n_blocks)).astype(np.uint64)
    roots = np.frombuffer(b"".join(hashlib.sha256(b"intake-block%d/%d" % (seed, b)).digest() for b in range(n_blocks)),
                          dtype=np.uint8).reshape(n_blocks, 32).copy()
    return parent, slot, roots


def _layout(csize=CSIZE, n_c=N_C):
    return (np.arange(n_c + 1) * csize).astype(np.uint32)


def _wire(wires):
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    return b"".join(wires), woff


def _oracle(wires, off, tree, epoch=EPOCH, current_slot=None, bits_stride=1):
    current_slot = (epoch + 1) * SPE + 1 if current_slot is None else current_slot
    blocks, ids = IO.block_store(*tree)
    return IO.intake_plain(wires, off, epoch, current_slot, DOMAIN, CPS, SPE, bits_stride, blocks, ids)


def _assert_equal(got, want, max_votes):
    n_votes = int(want.vote_off[-1])
    assert np.array_equal(got.status, want.status), (got.status.tolist(), want.status.tolist())
    assert np.array_equal(got.vote, want.vote)
    assert np.array_equal(np.asarray(got.vote_off, dtype=np.int64), want.vote_off)
    assert np.array_equal(got.sigs, want.sigs)
    k = min(n_votes, max_votes)
    for f in FIELDS[4:]:
        assert np.array_equal(getattr(got, f)[:k], getattr(want, f)[:k]), f
        assert not np.asarray(getattr(got, f)[k:]).any(), f


def _dev(eng, wires, off, epoch, current_slot, max_votes, bits_stride=1, woff=None):
    """Engine.attestation_intake_dev on device tensors; the results as numpy arrays"""
    dev = torch.device("cuda", 0)
    wire, w_off = _wire(wires)
    woff = w_off if woff is None else woff
    d_wire = torch.as_tensor(np.frombuffer(wire, dtype=np.uint8).copy(), device=dev)
    d_woff = torch.as_tensor(woff.view(np.int32), device=dev)
    d_off = torch.as_tensor(np.asarray(off, dtype=np.uint32).view(np.int32), device=dev)
    n_sig, n_c = int(off[-1]), len(off) - 1
    z = lambda *s, dt=torch.uint8: torch.zeros(s, dtype=dt, device=dev)      # noqa: E731
    out = [z(len(wires), dt=torch.int32), torch.full((n_sig,), -1, dtype=torch.int32, device=dev), z(n_c + 1, dt=torch.int32), z(n_sig, 96),
           z(max_votes, 128), z(max_votes, 32), z(max_votes, dt=torch.int64), z(max_votes, dt=torch.int64), z(max_votes, dt=torch.int32)]
    eng.attestation_intake_dev(d_wire, d_woff, d_off, epoch, current_slot, DOMAIN, CPS, SPE, bits_stride, *out)
    torch.cuda.synchronize()
    a = [x.cpu().numpy() for x in out]
    from pos_evolution_b200.engine import IntakeResult
    return IntakeResult(a[0], a[1].view(np.uint32), a[2].view(np.uint32), a[3], a[4], a[5], a[6].view(np.uint64), a[7].view(np.uint64),
                        a[8].view(np.uint32))


# ------------------------------------------------------------------------------------------ every status, every output
def _every_status_case(tree):
    """one or more attestations for each status 0-13 (the comment names it), in committees of CSIZE, plus duplicates"""
    parent, slot, roots = tree
    start = EPOCH * SPE
    R = lambda b: bytes(roots[b])      # noqa: E731
    # block 6 has slot start (24): the target of every head at or below it on its chain
    assert int(slot[6]) == start
    anc = lambda b: IO.ancestor(parent, slot, b, start)      # noqa: E731
    heads = [b for b in range(len(parent)) if int(slot[b]) <= start + 3 and anc(b) is not None]
    h1, h2 = heads[-1], heads[-2]

    def data(c, head, target=None, slot_=None, index=None, tepoch=EPOCH, src=0):
        s = start + c // CPS if slot_ is None else slot_
        t = R(anc(head)) if target is None else target
        return IO.data128(s, c % CPS if index is None else index, R(head), EPOCH - 1, R(src), tepoch, t)

    one = lambda p, n=CSIZE: [j == p for j in range(n)]      # noqa: E731
    sig = lambda k: hashlib.sha256(b"sig%d" % k).digest() * 3      # noqa: E731
    c = 6                                                            # slot start + 3
    A, Bd = data(c, h1), data(c, h2)
    w = []
    w.append(IO.encode(one(0), A, sig(0)))                            # 0
    w.append(IO.encode(one(1), Bd, sig(1)))                           # 0, another vote
    w.append(IO.encode(one(2), A, sig(2)))                            # 0, the first vote again
    w.append(IO.encode(one(0), A, sig(3)))                            # 13: duplicate, equal data
    w.append(IO.encode(one(1), A, sig(4)))                            # 13: duplicate, other data
    w.append(IO.encode(one(3), data(c, h1, target=R(0)), sig(5)))      # 12: target not the ancestor
    w.append(IO.encode(one(3), A, sig(6)))                            # 0: the earlier copy of position 3 failed
    w.append(IO.encode(one(4), A, sig(7))[:100])                      # 1: truncated container
    bad = bytearray(IO.encode(one(4), A, sig(8)))
    bad[0] = 229
    w.append(bytes(bad))                                              # 1: wrong offset
    bad = bytearray(IO.encode(one(4), A, sig(9)))
    bad[-1] = 0
    w.append(bytes(bad))                                              # 2: no delimiter
    w.append(IO.encode(one(4), A, sig(10))[:228])                     # 2: empty Bitlist
    w.append(IO.encode(one(0, 9), A, sig(11)))                        # 3: more bits than 8 * bits_stride
    w.append(IO.encode([True, True] + [False] * 5, A, sig(12)))       # 4: two bits
    w.append(IO.encode([False] * CSIZE, A, sig(13)))                  # 4: zero bits
    w.append(IO.encode(one(4, 6), A, sig(14)))                        # 5: wrong length
    w.append(IO.encode(one(4), data(c, h1, slot_=start + SPE), sig(15)))      # 6: foreign slot
    w.append(IO.encode(one(4), data(c, h1, slot_=start - 1), sig(16)))        # 6: foreign slot (the epoch before)
    w.append(IO.encode(one(4), data(c, h1, index=CPS), sig(17)))              # 6: foreign index
    w.append(IO.encode(one(4), data(c, h1, tepoch=EPOCH + 1), sig(18)))       # 7: wrong target epoch
    w.append(IO.encode(one(4), IO.data128(start + 7, 0, R(h1), EPOCH - 1, R(0), EPOCH, R(anc(h1))), sig(19)))  # 8 (current slot start + 7)
    w.append(IO.encode(one(4), data(c, h1)[:16] + bytes([7] * 32) + data(c, h1)[48:], sig(20)))     # 9: unknown head
    w.append(IO.encode(one(4), data(c, h1, target=bytes([9] * 32)), sig(21)))                      # 10: unknown target
    newer = next(b for b in range(len(parent)) if int(slot[b]) > start + 3 and anc(b) is not None)
    w.append(IO.encode(one(4), data(c, newer), sig(22)))               # 11: head newer than data.slot
    w.append(IO.encode(one(5), data(2, heads[0]), sig(24)))            # 0 in another committee
    return w


def test_every_status_and_output_matches_oracle(eng):
    tree = _tree()
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    wires = _every_status_case(tree)
    off = _layout()
    cur = EPOCH * SPE + 7
    want = _oracle(wires, off, tree, current_slot=cur)
    assert set(want.status.tolist()) == set(range(14)), sorted(set(want.status.tolist()))
    few = _oracle(wires[:3], off, tree, current_slot=cur)
    _assert_equal(_dev(eng, wires[:3], off, EPOCH, cur, 64), few, 64)
    wire, woff = _wire(wires)
    got = eng.attestation_intake(wire, woff, off, EPOCH, cur, DOMAIN, CPS, SPE, 1, 64)
    _assert_equal(got, want, 64)
    _assert_equal(_dev(eng, wires, off, EPOCH, cur, 64), want, 64)
    # the short list again, on the scratch the full one grew
    _assert_equal(_dev(eng, wires[:3], off, EPOCH, cur, 64), few, 64)
    assert eng.guard_flags() == 0


@pytest.mark.parametrize("seed", range(4))
def test_random_epochs_match_oracle(eng, seed):
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, 60, EPOCH * SPE - 7)
    eng.tree_load(*tree, np.ones(60, np.uint8))
    wires = IO.random_epoch(rng, EPOCH, SPE, CPS, CSIZE, tree, n_extra=30, corrupt=0.3, heads_per_committee=3)
    order = rng.permutation(len(wires))
    wires = [wires[i] for i in order]
    off = _layout()
    want = _oracle(wires, off, tree)
    got = eng.attestation_intake(*_wire(wires), off, EPOCH, (EPOCH + 1) * SPE + 1, DOMAIN, CPS, SPE, 1, 3 * N_C)
    _assert_equal(got, want, 3 * N_C)


def test_max_votes_overflow_is_refused(eng):
    from pos_evolution_b200.epoch import EpochProcessor
    tree = _tree()
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    rng = np.random.default_rng(7)
    wires = IO.random_epoch(rng, EPOCH, SPE, CPS, CSIZE, tree, corrupt=0.0, heads_per_committee=3)
    off = _layout()
    want = _oracle(wires, off, tree)
    n_votes = int(want.vote_off[-1])
    assert n_votes > N_C + 4
    mv = N_C + 4
    got = eng.attestation_intake(*_wire(wires), off, EPOCH, (EPOCH + 1) * SPE + 1, DOMAIN, CPS, SPE, 1, mv)
    _assert_equal(got, want, mv)            # the true counts in vote_off, the first max_votes rows
    n_val = int(off[-1])
    eng.registry_load(np.frombuffer(b"".join(scenarios.pubkeys(n_val)), dtype=np.uint8), np.full(n_val, 32 * 10**9, np.uint64))
    ep = EpochProcessor(eng, N_C, n_val, 1, len(tree[0]), device=torch.device("cuda", 0), max_votes=mv)
    ep.set_committees(np.arange(n_val, dtype=np.uint32), off)
    wire, woff = _wire(wires)
    dev = torch.device("cuda", 0)
    r = ep.intake_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=dev), torch.as_tensor(woff.view(np.int32), device=dev),
                      EPOCH, (EPOCH + 1) * SPE + 1, DOMAIN, CPS, SPE)
    assert np.array_equal(r.vote_off, want.vote_off)
    with pytest.raises(ValueError, match="max_votes"):
        ep.submit_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, votes=(r.vote, r.vote_off))
    assert not ep._inflight


# ------------------------------------------------------------------------------------------ end to end through the vote form
E2E_CPS, E2E_CSIZE = 1, 4
E2E_NC = SPE * E2E_CPS


def _e2e_epoch(eng, k, tree, members, off):
    """epoch EPOCH + k: every committee splits over 1-3 heads; about one member in five does not attest; committee 1's first member
    signs with a foreign key (its vote fails as a whole)"""
    parent, slot, roots = tree
    rng = np.random.default_rng(300 + k)
    e = EPOCH + k
    start = e * SPE
    wires, msgs, sks, who = [], [], [], []
    for c in range(E2E_NC):
        s = start + c
        ok = [b for b in range(len(parent)) if int(slot[b]) <= s and IO.ancestor(parent, slot, b, start) is not None]
        heads = [ok[int(i)] for i in rng.integers(0, len(ok), size=int(rng.integers(1, 4)))]
        for p in range(E2E_CSIZE):
            if rng.random() < 0.2 and not (c == 1 and p == 0):
                continue
            h = heads[int(rng.integers(0, len(heads)))]
            d = IO.data128(s, 0, bytes(roots[h]), e - 1, bytes(roots[0]), e, bytes(roots[IO.ancestor(parent, slot, h, start)]))
            msgs.append(_signing_root(d))
            v = int(members[off[c] + p])
            sks.append(scenarios.secret_key((v + 1) % len(members) if (c == 1 and p == 0) else v))
            bits = [j == p for j in range(E2E_CSIZE)]
            wires.append((bits, d))
    sig = eng.sign(sks, np.arange(len(msgs), dtype=np.uint32), np.frombuffer(b"".join(msgs), dtype=np.uint8).reshape(-1, 32))
    order = rng.permutation(len(wires))
    return [IO.encode(wires[i][0], wires[i][1], bytes(sig[i])) for i in order], e


def _signing_root(d):
    from oracle.spec import Spec
    return Spec.compute_signing_root(IO.data_from_bytes(d), DOMAIN)


_E2E = {}


def _e2e_expected(pks, members, off, tree, eff, epochs):
    """per epoch: oracle intake, and per vote the oracle's aggregate, verdict, aggregation_bits; heads after each epoch"""
    key = len(epochs)
    if key in _E2E:
        return _E2E[key]
    parent, slot, roots = tree
    m_epoch, m_block, m_has = np.zeros(len(members), np.uint64), np.zeros(len(members), np.uint32), np.zeros(len(members), np.uint8)
    equiv, active = np.zeros(len(members), np.uint8), np.ones(len(members), np.uint8)
    out = []
    for wires, e in epochs:
        blocks, ids = IO.block_store(*tree)
        r = IO.intake_plain(wires, off, e, (e + 1) * SPE, DOMAIN, E2E_CPS, SPE, 1, blocks, ids)
        aggs, oks, rows = [], [], []
        for v in range(int(r.vote_off[-1])):
            pos = np.nonzero(r.vote == v)[0]
            seg = [bytes(r.sigs[j]) for j in pos]
            agg = B.Aggregate(seg) if seg else bytes(96)
            ok = int(bool(seg) and B.FastAggregateVerify([pks[int(members[j])] for j in pos], bytes(r.msgs[v]), agg))
            aggs.append(agg)
            oks.append(ok)
            row = 0
            for j in pos:
                row |= 1 << int(j - off[np.searchsorted(off, j, side="right") - 1])
            rows.append(row)
            if ok:
                fast.lmd_update(m_epoch, m_block, m_has, equiv, [int(members[j]) for j in pos], int(r.target_epoch[v]), int(r.block_idx[v]))
        w = fast.ghost_weights(parent, m_block, m_has, eff, active, equiv, -1, 0)
        head = fast.ghost_head(parent, roots, fast.ghost_viable(parent, np.ones(len(parent), np.uint8)), w, 0)
        out.append((r, aggs, oks, rows, head))
    _E2E[key] = out
    return out


@pytest.mark.parametrize("mode", ["sync", "pipelined", "slasher"])
def test_end_to_end_matches_oracle_and_oracle_built_votes(eng, mode):
    from pos_evolution_b200.epoch import EpochProcessor, Intake
    tree = _tree(seed=3, n_blocks=40, first_slot=EPOCH * SPE - 5)
    n_val = E2E_NC * E2E_CSIZE
    pks = scenarios.pubkeys(n_val)
    members = np.random.default_rng(9).permutation(n_val).astype(np.uint32)
    off = _layout(E2E_CSIZE, E2E_NC)
    eff = np.full(n_val, 32 * 10**9, np.uint64)
    dev = torch.device("cuda", 0)
    epochs = [_e2e_epoch(eng, k, tree, members, off) for k in range(3)]
    want = _e2e_expected(pks, members, off, tree, eff, epochs)

    def run(feed):
        eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
        eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
        eng.latest_messages_reset()
        ep = EpochProcessor(eng, E2E_NC, n_val, 1, len(tree[0]), device=dev, depth=3, max_votes=3 * E2E_NC)
        ep.set_committees(members, off)
        if mode == "slasher":
            ep.enable_slasher(8, current_epoch=EPOCH, discount=True)
        side = torch.cuda.Stream()
        got, keep = [], []

        def collect(t):
            ok, hd = t.wait()
            found = t.slashings() if mode == "slasher" else None
            got.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().copy(), t.aggregation_bits().cpu().numpy().copy(),
                        None if found is None else (found.aggregate.tolist(), found.validator.tolist(), t.discounted().tolist())))
        for k, (wires, e) in enumerate(epochs):
            wire, woff = _wire(wires)
            if feed == "intake":
                with torch.cuda.stream(side):
                    r = ep.intake_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=dev), torch.as_tensor(woff.view(np.int32), device=dev),
                                      e, (e + 1) * SPE, DOMAIN, E2E_CPS, SPE)
                assert np.array_equal(r.status.cpu().numpy(), want[k][0].status)
            else:
                o, t = want[k][0], (lambda x: torch.as_tensor(x, device=dev))      # noqa: E731
                r = Intake(t(o.sigs), t(o.vote.view(np.int32)), t(o.msgs), t(o.target_epoch.view(np.int64)), t(o.block_idx.view(np.int32)),
                           t(o.source_epoch.view(np.int64)), t(o.data128), None, o.vote_off)
            keep.append(r)
            sl = dict(source_epoch=r.source_epoch, current_epoch=e) if mode == "slasher" else {}
            if mode == "sync":
                ok, hd = ep.process_epoch_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, votes=(r.vote, r.vote_off))
                s = ep.slots[0]
                n = int(r.vote_off[-1])
                got.append((ok.cpu().numpy().tolist(), int(hd.item()), s.agg_sig[:n].cpu().numpy().copy(), s.v_aggbits[:n].cpu().numpy().copy(), None))
            else:
                t = ep.submit_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, last=(k == len(epochs) - 1), votes=(r.vote, r.vote_off), **sl)
                if t is not None:
                    collect(t)
        if mode != "sync":
            for t in ep.drain():
                collect(t)
        assert eng.guard_flags() == 0
        return got

    got = run("intake")
    for k, (r, aggs, oks, rows, head) in enumerate(want):
        g_ok, g_head, g_agg, g_rows, _ = got[k]
        assert g_ok == oks, k
        assert g_head == head, k
        assert [bytes(a) for a in g_agg] == aggs, k
        assert [int(x[0]) for x in g_rows] == rows, k
    assert 0 in want[0][2] and 1 in want[0][2]
    # the same epochs fed the oracle's vote form: the same verdicts, heads, aggregates, bit rows (and slashings, discounted validators)
    ref = run("oracle")
    assert len(ref) == len(got)
    for x, y in zip(got, ref):
        assert x[0] == y[0] and x[1] == y[1] and np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3]) and x[4] == y[4]


# ------------------------------------------------------------------------------------------ the slot column follows prune and add
def test_tree_statuses_after_prune_and_add(eng):
    parent, slot, roots = _tree(seed=5, n_blocks=40, first_slot=EPOCH * SPE - 12)
    eng.tree_load(parent, slot, roots, np.ones(40, np.uint8))
    keep_root = 4
    m = eng.tree_prune(keep_root)
    p2, s2, r2 = _pruned((parent, slot, roots), m)
    # two new blocks: one under the newest kept block, one that forks at slot start
    n2 = len(p2)
    last = int(np.argmax(s2))
    add_p = np.array([last, int(np.nonzero(s2 <= EPOCH * SPE)[0][-1])], dtype=np.uint32)
    add_s = np.array([int(s2[last]) + 1, EPOCH * SPE + 2], dtype=np.uint64)
    add_r = np.frombuffer(hashlib.sha256(b"added0").digest() + hashlib.sha256(b"added1").digest(), dtype=np.uint8).reshape(2, 32)
    eng.tree_add(add_p, add_s, add_r, np.ones(2, np.uint8))
    tree = (np.concatenate([p2, add_p]), np.concatenate([s2, add_s]), np.vstack([r2, add_r]))
    assert eng.tree_size() == n2 + 2
    rng = np.random.default_rng(11)
    wires = IO.random_epoch(rng, EPOCH, SPE, CPS, CSIZE, tree, n_extra=10, corrupt=0.3, heads_per_committee=3)
    # and attestations whose roots are blocks the prune dropped
    dropped = np.nonzero(m == 0xFFFFFFFF)[0]
    for j, b in enumerate(dropped[:4]):
        d = IO.data128(EPOCH * SPE + 2, 0, bytes(roots[b]) if j % 2 == 0 else bytes(tree[2][0]), EPOCH - 1, bytes(32), EPOCH,
                       bytes(roots[b]) if j % 2 else bytes(tree[2][0]))
        wires.append(IO.encode([i == j for i in range(CSIZE)], d, bytes(96)))
    off = _layout()
    want = _oracle(wires, off, tree)
    assert {9, 10} <= set(want.status.tolist()) and 0 in want.status
    got = eng.attestation_intake(*_wire(wires), off, EPOCH, (EPOCH + 1) * SPE + 1, DOMAIN, CPS, SPE, 1, 3 * N_C)
    _assert_equal(got, want, 3 * N_C)
    # pruned to a block above start_slot(e): a walk from a head reaches the tree's root still above it (status 12)
    above = int(np.nonzero(tree[1] > EPOCH * SPE)[0][0])
    tree = _pruned(tree, eng.tree_prune(above))
    assert int(tree[1][0]) <= EPOCH * SPE + 7
    wires = wires + [IO.encode([i == 6 for i in range(CSIZE)], IO.data128(EPOCH * SPE + 7, 0, bytes(tree[2][0]), EPOCH - 1, bytes(32), EPOCH,
                                                                        bytes(tree[2][0])), bytes(96))]
    want = _oracle(wires, off, tree)
    assert want.status[-1] == 12
    got = eng.attestation_intake(*_wire(wires), off, EPOCH, (EPOCH + 1) * SPE + 1, DOMAIN, CPS, SPE, 1, 3 * N_C)
    _assert_equal(got, want, 3 * N_C)


def _pruned(tree, m):
    """the host arrays of the tree after a prune with map m"""
    parent, slot, roots = tree
    old = np.nonzero(m != 0xFFFFFFFF)[0]
    old = old[np.argsort(m[old])]
    return (np.array([0] + [int(m[parent[b]]) for b in old[1:]], dtype=np.uint32), slot[old].copy(), roots[old].copy())


# ------------------------------------------------------------------------------------------ error contract of the host form
def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _raw_call(e, wire, woff, off, epoch, current_slot, n_c=N_C, mv=16):
    n_att, n_sig = len(woff) - 1, int(off[-1])
    outs = [np.full(sz, SENTINEL, np.uint8) for sz in (4 * n_att, 4 * n_sig, 4 * (N_C + 1), 96 * n_sig, 128 * mv, 32 * mv, 8 * mv, 8 * mv, 4 * mv)]
    w = np.frombuffer(wire, np.uint8)
    rc = e.lib.b2_attestation_intake(e.h, _p(w), len(wire), _p(np.asarray(woff, np.uint32)), n_att, _p(np.asarray(off, np.uint32)), n_c, CPS, SPE, 1,
                                     epoch, current_slot, _p(np.frombuffer(DOMAIN, np.uint8)), mv, *[_p(o) for o in outs])
    return rc, outs


def test_rejected_host_calls_change_nothing(eng):
    from pos_evolution_b200 import _lib
    from pos_evolution_b200.engine import Engine
    tree = _tree()
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    wires = _every_status_case(tree)
    wire, woff = _wire(wires)
    off = _layout()
    cur = (EPOCH + 1) * SPE + 1
    weights, head = eng.get_weights(), eng.get_head(0)
    rc, _ = _raw_call(eng, wire, woff, off, EPOCH, cur)
    assert rc == 0
    bad_woff = woff.copy()
    bad_woff[3], bad_woff[4] = bad_woff[4], bad_woff[3]
    past = woff.copy()
    past[-1] += 1
    cases = [(wire, bad_woff, off, EPOCH, cur, N_C), (wire, past, off, EPOCH, cur, N_C), (wire, woff, off, EPOCH, cur, N_C - 1),
             (wire, woff, off, EPOCH + 2, cur, N_C), (wire, woff, off, EPOCH - 1, cur, N_C), (wire, woff, off, EPOCH, cur + 100, N_C)]
    for wr, wo, of, e, c, n_c in cases:
        o = of[:n_c + 1]
        rc, outs = _raw_call(eng, wr, wo, o, e, c, n_c=n_c)
        assert rc == _lib.B2_EINVAL
        assert all((x == SENTINEL).all() for x in outs)
    assert np.array_equal(eng.get_weights(), weights) and eng.get_head(0) == head and eng.tree_size() == len(tree[0])
    fresh = Engine(0)      # no tree
    try:
        rc, outs = _raw_call(fresh, wire, woff, off, EPOCH, cur)
        assert rc == _lib.B2_EINVAL and all((x == SENTINEL).all() for x in outs)
    finally:
        fresh.close()


# ------------------------------------------------------------------------------------------ device guards
def test_device_guards(eng):
    tree = _tree()
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    wires = _every_status_case(tree)
    off = _layout()
    cur = EPOCH * SPE + 7
    want = _oracle(wires, off, tree, current_slot=cur)
    assert eng.guard_flags() == 0
    # a reversed woff row and one that ends past the wire: status 1 for those two attestations, everything else as before
    wire, woff = _wire(wires)
    woff = woff.copy()
    woff[1] = woff[2] + 1                     # row 0 ends after row 1 ends: row 1 reversed
    got = _dev(eng, wires, off, EPOCH, cur, 64, woff=woff)
    assert eng.guard_flags() & 2 and got.status[1] == 1
    woff2 = _wire(wires)[1].copy()
    woff2[-1] = len(wire) + 64
    got = _dev(eng, wires, off, EPOCH, cur, 64, woff=woff2)
    assert eng.guard_flags() & 2 and got.status[-1] == 1
    assert np.array_equal(got.status[:-1], want.status[:-1])
    # a malformed committee row: committee 6 ends past n_sig -> only its placeholder, its attestations status 5
    bad = off.copy().astype(np.int64)
    bad[7] = bad[-1] + 5
    got = _dev(eng, wires, bad.astype(np.uint32), EPOCH, cur, 64)
    assert eng.guard_flags() & 2
    c6 = [i for i, w in enumerate(wires) if want.status[i] in (0, 13) and int.from_bytes(w[4:12], "little") == EPOCH * SPE + 3]
    assert c6 and all(got.status[i] == 5 for i in c6)
    assert int(got.vote_off[7]) - int(got.vote_off[6]) == 1


# ------------------------------------------------------------------------------------------ full size
def test_full_size_epoch_matches_numpy_oracle(eng):
    spe, cps, csize, epoch = 32, 64, 512, 5
    n_c = spe * cps
    n = n_c * csize
    rng = np.random.default_rng(2024)
    nb = 64
    parent = np.array([0] + [max(0, b - 1 - int(rng.integers(0, 2))) for b in range(1, nb)], dtype=np.uint32)
    slot = (epoch * spe - 20 + np.arange(nb)).astype(np.uint64)
    roots = np.frombuffer(b"".join(hashlib.sha256(b"full%d" % b).digest() for b in range(nb)), np.uint8).reshape(nb, 32).copy()
    eng.tree_load(parent, slot, roots, np.ones(nb, np.uint8))
    start = epoch * spe
    L = 228 + csize // 8 + 1
    c = np.repeat(np.arange(n_c), csize)
    p = np.tile(np.arange(csize), n_c)
    # two heads per committee, among the blocks at or before its slot
    s_c = start + np.arange(n_c) // cps
    data = np.zeros((n_c, 2, 128), np.uint8)
    for k in range(n_c):
        ok = np.nonzero(slot <= s_c[k])[0]
        for v in range(2):
            h = int(ok[rng.integers(0, len(ok))])
            t = IO.ancestor(parent, slot, h, start)
            data[k, v] = np.frombuffer(IO.data128(int(s_c[k]), k % cps, bytes(roots[h]), epoch - 1, bytes(roots[0]), epoch, bytes(roots[t])), np.uint8)
    rec = np.zeros((n, L), np.uint8)
    rec[:, 0] = 228
    rec[:, 4:132] = data[c, rng.integers(0, 2, size=n)]
    rec[:, 132:228] = rng.integers(0, 256, size=(n, 96), dtype=np.uint8)
    rec[np.arange(n), 228 + p // 8] = (1 << (p % 8)).astype(np.uint8)
    rec[:, L - 1] |= 1      # the delimiter: bit 512 = bit 0 of byte 64
    unknown = rng.choice(n, size=300, replace=False)
    rec[unknown, 20:52] = rng.integers(0, 256, size=(300, 32), dtype=np.uint8)
    dup = rng.choice(n, size=n // 100, replace=False)
    extra = rec[dup].copy()
    extra[::2, 4 + 56] ^= 1      # half of the duplicates carry other data
    rec = np.vstack([rec, extra])
    rec = rec[rng.permutation(rec.shape[0])]
    off = (np.arange(n_c + 1) * csize).astype(np.uint32)
    cur = (epoch + 1) * spe + 3
    mv = 2 * n_c + 64
    want = IO.intake_numpy(rec, off.astype(np.int64), epoch, cur, DOMAIN, cps, spe, csize // 8, parent, slot, roots)
    assert {0, 9, 13} <= set(want.status.tolist())
    woff = (np.arange(rec.shape[0] + 1, dtype=np.uint64) * L).astype(np.uint32)
    got = eng.attestation_intake(rec.tobytes(), woff, off, epoch, cur, DOMAIN, cps, spe, csize // 8, mv)
    _assert_equal(got, want, mv)
    assert eng.guard_flags() == 0
