"""GPU parity of the vote form of the epoch pipeline (EpochProcessor(..., max_votes=M), votes=(vote, vote_off); b2_votes_group_dev):
committees whose members signed different AttestationData, with non-attesters, a committee where nobody attested and a vote with a
foreign signature, against the oracle (bls.Aggregate / FastAggregateVerify per vote, update_latest_messages in vote order, get_head) in
every mode of test_gpu_epoch.py; equivalence with the committee form at one vote per committee; the device guards and the host
refusals; the slasher and the discount over split committees."""
import hashlib

import numpy as np
import pytest
import torch

import scenarios
from oracle import bls_sig as B
from oracle import fast

pytestmark = pytest.mark.gpu

N_VAL, CSIZE, N_C, N_BLK, N_EPOCHS = 48, 8, 6, 40, 4
NONE = 0xFFFFFFFF
PLACEHOLDER, FOREIGN = 4, 1            # the committee where nobody attests; the committee whose first vote carries a foreign signature
ZERO96 = bytes(96)


@pytest.fixture(scope="module")
def world():
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    pks = scenarios.pubkeys(N_VAL)
    rng = np.random.default_rng(5)
    members = rng.permutation(N_VAL).astype(np.uint32)
    off = (np.arange(N_C + 1) * CSIZE).astype(np.uint32)
    tree = scenarios.fork_tree(N_BLK, 5)
    eff = rng.integers(16, 33, size=N_VAL).astype(np.uint64) * np.uint64(10**9)
    yield eng, pks, members, off, tree, eff
    eng.close()


def _sign(eng, validators, msg_idx, msgs):
    return eng.sign([scenarios.secret_key(int(v)) for v in validators], np.asarray(msg_idx, dtype=np.uint32), msgs)


def _epoch(eng, k, members, off):
    """Inputs of epoch k: 1-3 votes per committee (committee PLACEHOLDER: one vote, nobody attests), ~15 % non-attesters, committee
    FOREIGN's first vote has one member's signature replaced by another validator's over the same message."""
    rng = np.random.default_rng(100 + k)
    nv = rng.integers(1, 4, size=N_C)
    nv[PLACEHOLDER], nv[FOREIGN] = 1, 2
    vote_off = np.concatenate([[0], np.cumsum(nv)]).astype(np.int64)
    n_votes = int(vote_off[-1])
    vote = np.full(N_VAL, NONE, dtype=np.int64)
    for c in range(N_C):
        if c == PLACEHOLDER:
            continue
        ids = vote_off[c] + rng.integers(0, nv[c], size=CSIZE)
        if c == FOREIGN:                                  # both votes attested, the first by positions 0..2
            ids = np.where(np.arange(CSIZE) < 3, vote_off[c], vote_off[c] + 1)
        absent = rng.random(CSIZE) < 0.15
        if c == FOREIGN:
            absent[[0, 1, 3]] = False
        vote[off[c]:off[c + 1]] = np.where(absent, NONE, ids)
    msgs = np.frombuffer(b"".join(hashlib.sha256(b"epoch%d/vote%d" % (k, v)).digest() for v in range(n_votes)), dtype=np.uint8).reshape(-1, 32)
    vote_of = np.where(vote == NONE, 0, vote)
    sigs = _sign(eng, members, vote_of, msgs)
    j = int(off[FOREIGN])                                 # position 0 of committee FOREIGN, vote vote_off[FOREIGN]
    sigs[j] = _sign(eng, [(int(members[j]) + 1) % N_VAL], [vote_off[FOREIGN]], msgs)[0]
    sigs[vote == NONE] = rng.integers(0, 256, size=(int((vote == NONE).sum()), 96), dtype=np.uint8)      # never read
    te = np.full(n_votes, 2 + k, dtype=np.int64)
    bi = rng.integers(0, N_BLK, size=n_votes).astype(np.int32)
    return dict(vote=vote.astype(np.uint32), vote_off=vote_off, msgs=msgs, sigs=sigs, te=te, bi=bi, n_votes=n_votes)


def _vote_members(E, members, off):
    """per vote: its committee positions and validators, in committee order"""
    out = []
    for c in range(N_C):
        for v in range(int(E["vote_off"][c]), int(E["vote_off"][c + 1])):
            pos = [j for j in range(CSIZE) if int(E["vote"][off[c] + j]) == v]
            out.append((c, pos, [int(members[off[c] + j]) for j in pos]))
    return out


_CACHE = {}


def _expected(pks, members, off, E, k):
    """oracle per vote: aggregate (96 zero bytes when nobody attested), verdict, aggregation_bits row"""
    if k not in _CACHE:
        aggs, oks, rows = [], [], []
        for v, (c, pos, vals) in enumerate(_vote_members(E, members, off)):
            seg = [bytes(E["sigs"][off[c] + j]) for j in pos]
            agg = B.Aggregate(seg) if seg else ZERO96
            aggs.append(agg)
            oks.append(int(bool(seg) and B.FastAggregateVerify([pks[x] for x in vals], bytes(E["msgs"][v]), agg)))
            row = np.zeros(1, dtype=np.uint8)
            for j in pos:
                row[0] |= 1 << j
            rows.append(row)
        _CACHE[k] = (aggs, oks, np.array(rows))
    return _CACHE[k]


MODES = [("sync", 3), ("pipelined", 2), ("pipelined", 3), ("pipelined", 4), ("pipelined", 8), ("pipelined", 12), ("pipelined_host", 3),
         ("pipelined_host", 2), ("sync_host", 3), ("pipelined_team", 6), ("sync_rlc", 3), ("pipelined_rlc", 3), ("pipelined_host_rlc", 4)]


@pytest.mark.parametrize("mode,depth", MODES)
def test_vote_form_matches_oracle(world, mode, depth):
    eng, pks, members, off, tree, eff = world
    from pos_evolution_b200.epoch import EpochProcessor
    rlc = mode.endswith("_rlc")
    mode = mode[:-4] if rlc else mode
    tail_form = "team" if mode == "pipelined_team" else "thread"
    mode = "pipelined" if mode == "pipelined_team" else mode
    parent, slot, roots, leaf_viable = tree
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(parent, slot, roots, leaf_viable)
    eng.latest_messages_reset()
    eng.set_verify_mode(rlc, hashlib.sha256(b"votes-seed").digest() if rlc else None)
    dev = torch.device("cuda", 0)
    ep = EpochProcessor(eng, N_C, N_VAL, 1, N_BLK, device=dev, depth=depth, tail_form=tail_form, max_votes=3 * N_C)
    ep.set_committees(members, off)
    m_epoch, m_block, m_has = np.zeros(N_VAL, np.uint64), np.zeros(N_VAL, np.uint32), np.zeros(N_VAL, np.uint8)
    equiv, active = np.zeros(N_VAL, np.uint8), np.ones(N_VAL, np.uint8)
    got, want, keep = [], [], []

    def collect(t):
        ok, hd = t.wait()
        got.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().copy(), t.aggregation_bits().cpu().numpy().copy(), None))

    for k in range(N_EPOCHS):
        E = _epoch(eng, k, members, off)
        aggs, oks, rows = _expected(pks, members, off, E, k)
        assert oks[int(E["vote_off"][FOREIGN])] == 0 and oks[int(E["vote_off"][FOREIGN]) + 1] == 1
        assert oks[int(E["vote_off"][PLACEHOLDER])] == 0 and aggs[int(E["vote_off"][PLACEHOLDER])] == ZERO96
        for v, (c, pos, vals) in enumerate(_vote_members(E, members, off)):
            if oks[v]:
                fast.lmd_update(m_epoch, m_block, m_has, equiv, vals, int(E["te"][v]), int(E["bi"][v]))
        w = fast.ghost_weights(parent, m_block, m_has, eff, active, equiv, -1, 0)
        head = fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0)
        want.append((oks, head, aggs, rows, (m_epoch.copy(), m_block.copy(), m_has.copy())))
        d = [torch.as_tensor(E["sigs"], device=dev), None, torch.as_tensor(E["msgs"], device=dev), torch.as_tensor(E["te"], device=dev),
             torch.as_tensor(E["bi"], device=dev)]
        dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
        keep.append((d, dv))
        if mode in ("pipelined_host", "sync_host"):
            h = [x.cpu().pin_memory() if x is not None else None for x in d]
            hv = dv.cpu().pin_memory()
            keep.append((h, hv))
            if mode == "sync_host":
                ok, hd = ep.process_epoch_host(*h, votes=(hv, E["vote_off"]))
                s = ep.slots[0]
                got.append((ok.numpy().tolist(), hd, s.h_agg_sig[:E["n_votes"]].numpy().copy(), s.h_aggbits[:E["n_votes"]].numpy().copy(),
                            eng.latest_messages_read()))
            else:
                t = ep.submit_host(*h, last=(k == N_EPOCHS - 1), votes=(hv, E["vote_off"]))
                if t is not None:
                    collect(t)
        elif mode == "sync":
            ok, hd = ep.process_epoch_dev(*d, votes=(dv, E["vote_off"]))
            torch.cuda.synchronize()
            s = ep.slots[0]
            got.append((ok.cpu().numpy().tolist(), int(hd.item()), s.agg_sig[:E["n_votes"]].cpu().numpy().copy(),
                        s.v_aggbits[:E["n_votes"]].cpu().numpy().copy(), eng.latest_messages_read()))
        else:
            t = ep.submit_dev(*d, last=(k % 3 == 2), votes=(dv, E["vote_off"]))
            if t is not None:
                collect(t)
    if mode in ("pipelined", "pipelined_host"):
        for t in ep.drain():
            collect(t)
    assert eng.guard_flags() == 0
    assert len(got) == N_EPOCHS
    for k in range(N_EPOCHS):
        oks, head, aggs, rows, lmd = want[k]
        g_ok, g_head, g_agg, g_rows, g_lmd = got[k]
        assert g_ok == oks, k
        assert g_head == head, k
        assert [bytes(r) for r in g_agg] == aggs, k
        assert np.array_equal(g_rows, rows), k
        if g_lmd is not None:                             # synchronous forms: the LMD table after every epoch
            e, b, h = g_lmd
            assert np.array_equal(h, lmd[2]) and np.array_equal(e[h == 1], lmd[0][h == 1]) and np.array_equal(b[h == 1], lmd[1][h == 1]), k
    e, b, h = eng.latest_messages_read()
    assert np.array_equal(h, m_has) and np.array_equal(e[h == 1], m_epoch[h == 1]) and np.array_equal(b[h == 1], m_block[h == 1])
    eng.set_verify_mode(False)


# ------------------------------------------------------------------------------------------ one vote per committee == committee form
def _single_vote_epochs(eng, members, off, participation, n_epochs=3):
    out = []
    for k in range(n_epochs):
        rng = np.random.default_rng(200 + k)
        msgs = np.frombuffer(b"".join(hashlib.sha256(b"single%d/%d" % (k, c)).digest() for c in range(N_C)), dtype=np.uint8).reshape(-1, 32)
        com = np.repeat(np.arange(N_C), CSIZE)
        sigs = _sign(eng, members, com, msgs)
        att = rng.random(N_VAL) < participation
        sigs[~att] = np.frombuffer(bytes([0xC0]) + bytes(95), dtype=np.uint8)       # the committee form's non-signer: the identity
        bits = np.zeros((N_C, 1), dtype=np.uint8)
        for i in np.nonzero(att)[0]:
            bits[i // CSIZE, 0] |= 1 << (i % CSIZE)
        if k == 1:
            sigs[3] = _sign(eng, [int(members[4])], [0], msgs)[0]                     # committee 0 fails (if position 3 attests)
        vote = np.where(att, com, NONE).astype(np.uint32)
        out.append(dict(msgs=msgs, sigs=sigs, bits=bits, vote=vote, te=np.full(N_C, 3 + k, dtype=np.int64),
                        bi=((np.arange(N_C) * 5 + k) % N_BLK).astype(np.int32)))
    return out


@pytest.mark.parametrize("participation", [1.0, 0.7])
def test_one_vote_per_committee_equals_committee_form(world, participation):
    eng0, pks, members, off, tree, eff = world
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    dev = torch.device("cuda", 0)
    epochs = _single_vote_epochs(eng0, members, off, participation)
    vote_off = np.arange(N_C + 1)
    res = []
    for votes in (False, True):
        eng = Engine(0)
        eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
        eng.tree_load(*tree)
        eng.latest_messages_reset()
        ep = EpochProcessor(eng, N_C, N_VAL, 1, N_BLK, device=dev, depth=3, max_votes=N_C if votes else None)
        ep.set_committees(members, off)
        out, keep = [], []
        for k, E in enumerate(epochs):
            d = [torch.as_tensor(E["sigs"], device=dev), torch.as_tensor(E["bits"], device=dev), torch.as_tensor(E["msgs"], device=dev),
                 torch.as_tensor(E["te"], device=dev), torch.as_tensor(E["bi"], device=dev)]
            dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
            keep.append((d, dv))
            if votes:
                d[1] = None
            t = ep.submit_dev(*d, last=k == len(epochs) - 1, votes=(dv, vote_off) if votes else None)
            for t in ([t] if t is not None else []) + (ep.drain() if k == len(epochs) - 1 else []):
                ok, hd = t.wait()
                out.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().tobytes()))
        res.append((out, eng.latest_messages_read()))
        assert eng.guard_flags() == 0
        eng.close()
    (a, la), (b, lb) = res
    assert a == b
    assert all(np.array_equal(x, y) for x, y in zip(la, lb))


# ------------------------------------------------------------------------------------------ guards and refusals
def _processor(world, max_votes=3 * N_C, depth=3):
    eng, pks, members, off, tree, eff = world
    from pos_evolution_b200.epoch import EpochProcessor
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(*tree)
    eng.latest_messages_reset()
    ep = EpochProcessor(eng, N_C, N_VAL, 1, N_BLK, device=torch.device("cuda", 0), depth=depth, max_votes=max_votes)
    ep.set_committees(members, off)
    return ep


def _run_sync(ep, E):
    dev = torch.device("cuda", 0)
    d = [torch.as_tensor(E["sigs"], device=dev), None, torch.as_tensor(E["msgs"], device=dev), torch.as_tensor(E["te"], device=dev),
         torch.as_tensor(E["bi"], device=dev)]
    ok, hd = ep.process_epoch_dev(*d, votes=(torch.as_tensor(E["vote"].view(np.int32), device=dev), E["vote_off"]))
    torch.cuda.synchronize()
    s = ep.slots[0]
    return ok.cpu().numpy().tolist(), int(hd.item()), s.agg_sig[:E["n_votes"]].cpu().numpy().copy(), s.v_aggbits[:E["n_votes"]].cpu().numpy().copy()


def test_vote_id_outside_its_committee_is_skipped_and_reported(world):
    eng, pks, members, off, tree, eff = world
    E = _epoch(eng, 0, members, off)
    # committee 0's attesters: one names a vote of committee 2, one an id past n_votes -- both count as not attesting
    c0 = [j for j in range(CSIZE) if E["vote"][j] != NONE]
    bad = dict(E, vote=E["vote"].copy())
    bad["vote"][c0[0]] = E["vote_off"][2]
    bad["vote"][c0[1]] = 10**6
    ref = dict(E, vote=E["vote"].copy())
    ref["vote"][c0[:2]] = NONE
    ep = _processor(world)
    got = _run_sync(ep, bad)
    assert eng.guard_flags() & 1                     # B2_GUARD_BAD_INDEX
    ep = _processor(world)
    exp = _run_sync(ep, ref)
    assert eng.guard_flags() == 0
    assert got[0] == exp[0] and got[1] == exp[1] and np.array_equal(got[2], exp[2]) and np.array_equal(got[3], exp[3])


def test_malformed_vote_off_on_the_device_empties_every_vote(world):
    eng, pks, members, off, tree, eff = world
    dev = torch.device("cuda", 0)
    _processor(world)
    E = _epoch(eng, 0, members, off)
    nv = E["n_votes"]
    vo = E["vote_off"].astype(np.int32).copy()
    vo[2] = vo[1]                                    # committee 1 without a vote id
    t = lambda a, dt=torch.int32: torch.as_tensor(np.ascontiguousarray(a), device=dev).to(dt)      # noqa: E731
    seg, bits, agg = t(np.full(nv + 1, 7)), torch.full((nv, 1), 0xAB, dtype=torch.uint8, device=dev), torch.zeros((nv, 1), dtype=torch.uint8, device=dev)
    sig_out, mem_out, pos_out = torch.zeros((N_VAL, 96), dtype=torch.uint8, device=dev), t(np.zeros(N_VAL)), t(np.zeros(N_VAL))
    eng.votes_group_dev(t(E["vote"].view(np.int32)), t(vo), t(members.view(np.int32)), t(off.view(np.int32)), t(E["sigs"], torch.uint8), 0, N_C,
                        sig_out, mem_out, pos_out, seg, bits, agg)
    assert eng.guard_flags() & 2                     # B2_GUARD_BAD_ROW
    assert seg.cpu().numpy().tolist() == [0] * (nv + 1) and not bits.any() and not agg.any()


def test_refusals_before_anything_is_enqueued(world):
    eng, pks, members, off, tree, eff = world
    dev = torch.device("cuda", 0)
    E = _epoch(eng, 0, members, off)
    d = [torch.as_tensor(E["sigs"], device=dev), None, torch.as_tensor(E["msgs"], device=dev), torch.as_tensor(E["te"], device=dev),
         torch.as_tensor(E["bi"], device=dev)]
    dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
    small = _processor(world, max_votes=E["n_votes"] - 1)
    plain = _processor(world, max_votes=None)
    ep = _processor(world)
    bad_offs = [E["vote_off"][:-1], np.concatenate([[1], E["vote_off"][1:]]), np.where(np.arange(N_C + 1) == 2, E["vote_off"][1], E["vote_off"]),
                np.concatenate([[0], np.full(N_C, 9)])]
    n0, k0 = eng.launch_count, ep.k
    for vo in bad_offs:
        for call in (ep.process_epoch_dev, ep.submit_dev):
            with pytest.raises(ValueError):
                call(*d, votes=(dv, vo))
    with pytest.raises(ValueError):
        small.submit_dev(*d, votes=(dv, E["vote_off"]))
    with pytest.raises(ValueError):
        plain.process_epoch_dev(*d, votes=(dv, E["vote_off"]))
    torch.cuda.synchronize()
    assert eng.launch_count == n0 and ep.k == k0 and not ep._inflight and small.k == plain.k == 0


# ------------------------------------------------------------------------------------------ slasher + discount
@pytest.mark.parametrize("pipelined", [False, True])
def test_slasher_and_discount_name_votes_and_committee_positions(world, pipelined):
    """Two epochs with the same target and other votes: every member accepted in both double-votes.  The flagged slots name the second
    epoch's vote ids and committee positions; the discount marks exactly those validators."""
    eng, pks, members, off, tree, eff = world
    dev = torch.device("cuda", 0)
    ep = _processor(world)
    ep.enable_slasher(8, current_epoch=3, discount=True)
    E0, E1 = _epoch(eng, 0, members, off), _epoch(eng, 1, members, off)
    for E in (E0, E1):
        E["te"][:] = 3
    first = {}                                        # validator -> root of its accepted vote in epoch 0
    want = []
    for i, E in enumerate((E0, E1)):
        aggs, oks, rows = _expected(pks, members, off, E, i)
        for v, (c, pos, vals) in enumerate(_vote_members(E, members, off)):
            if not oks[v]:
                continue
            for j, x in zip(pos, vals):
                if i == 0:
                    first[x] = bytes(E["msgs"][v])
                elif x in first and first[x] != bytes(E["msgs"][v]):
                    want.append((v, j, x))
    assert want
    tickets, keep = [], []
    for k, E in enumerate((E0, E1)):
        d = [torch.as_tensor(E["sigs"], device=dev), None, torch.as_tensor(E["msgs"], device=dev), torch.as_tensor(E["te"], device=dev),
             torch.as_tensor(E["bi"], device=dev)]
        src = torch.zeros(E["n_votes"], dtype=torch.int64, device=dev)
        dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
        keep.append((d, src, dv))
        if pipelined:
            t = ep.submit_dev(*d, votes=(dv, E["vote_off"]), source_epoch=src, current_epoch=3, last=k == 1)
            tickets += [t] if t is not None else []
        else:
            ep.process_epoch_dev(*d, votes=(dv, E["vote_off"]), source_epoch=src, current_epoch=3)
            torch.cuda.synchronize()
            tickets.append(None)
            if k == 0:
                assert len(ep.slashings().validator) == 0
    if pipelined:
        tickets += ep.drain()
        assert len(tickets[0].slashings().validator) == 0
        sl, disc = tickets[1].slashings(), tickets[1].discounted()
    else:
        sl, disc = ep.slashings(), ep.discounted()
    got = sorted(zip(sl.aggregate.tolist(), sl.position.tolist(), sl.validator.tolist()))
    assert got == sorted(want)
    assert set(sl.kind.tolist()) == {1}
    assert disc.tolist() == sorted({x for _, _, x in want})
    assert np.nonzero(ep.equivocating())[0].tolist() == disc.tolist()
