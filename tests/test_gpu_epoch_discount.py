"""Equivocation discounting inside the epoch pipeline (EpochProcessor.enable_slasher(..., discount=True), pos-evolution.md:1405-1461) on
the six-epoch world and planted offences of test_gpu_epoch_slasher.py.  The sequential oracle, per epoch k in submission order, with
one set E of equivocating validators:
  1. update_latest_messages (:1435-1441) for the accepted aggregates of k, in aggregate order, skipping members in E;
  2. head_k = get_head counting no validator in E;
  3. the slasher update of epoch k (tests/slasher_oracle.BruteSlasher);
  4. E |= every validator with a flagged member slot of epoch k.
Every mode must match it: heads, the newly discounted validators of each epoch, and after drain() the equivocating and LMD tables;
verdicts and aggregate signatures must equal a run with discounting off.  Also: a planted balancing pattern whose head moves only with
discounting on, validators marked before the run, the range form over the golden streams, and the C ABI's error contract."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import scenarios
import slasher_oracle as SO
import test_gpu_epoch_slasher as T
from oracle import fast

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _oracle(epochs, members, off, tree, eff, n_val, H, pre_marked=(), n_epochs=None):
    """the sequence above -> per epoch (head, sorted newly discounted validators), then the final (E, epoch, block, has_msg)"""
    parent, slot, roots, leaf_viable = tree
    m_epoch, m_block, m_has = np.zeros(n_val, np.uint64), np.zeros(n_val, np.uint32), np.zeros(n_val, np.uint8)
    equiv, active = np.zeros(n_val, np.uint8), np.ones(n_val, np.uint8)
    equiv[list(pre_marked)] = 1
    bs = SO.BruteSlasher(n_val, H, 2 * (len(off) - 1), T.CUR0)
    out = []
    for k, e in enumerate(epochs[:n_epochs]):
        n_agg = len(off) - 1
        for a in range(n_agg):
            if e["ok"][a]:
                sel = [int(members[off[a] + j]) for j in range(off[a + 1] - off[a]) if (e["bits"][a, j >> 3] >> (j & 7)) & 1]
                fast.lmd_update(m_epoch, m_block, m_has, equiv, sel, int(e["tgt"][a]), int(e["blk"][a]))
        w = fast.ghost_weights(parent, m_block, m_has, eff, active, equiv, -1, 0)
        head = fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0)
        bs.advance(T.CUR0 + k)
        _, kind, _, _ = bs.update(members, off, e["bits"], e["src"].astype(np.uint64), e["tgt"].astype(np.uint64), e["msgs"], e["ok"])
        flagged = np.unique(members[:len(kind)][kind != 0].astype(np.int64))
        new = flagged[equiv[flagged] == 0]
        equiv[flagged] = 1
        out.append((head, new))
    m_block[m_has == 0] = 0
    return out, (equiv, m_epoch, m_block, m_has)


def _run(eng, epochs, members, off, n_blk, mode, depth, H, discount, n_agg=T.N_AGG, csize=T.CSIZE):
    """epochs through EpochProcessor in `mode` -> per epoch (verdicts, head, aggregate signatures, kind, discounted or None), then the
    final (equivocating, epoch, block, has_msg) tables"""
    from pos_evolution_b200.epoch import EpochProcessor
    dev = torch.device("cuda", 0)
    ep = EpochProcessor(eng, n_agg, n_agg * csize, epochs[0]["bits"].shape[1], n_blk, device=dev, depth=depth, tail_form="thread")
    ep.set_committees(members, off)
    ep.enable_slasher(H, current_epoch=T.CUR0, discount=discount)
    results, keep = [], []

    def collect(t):
        ok, hd = t.wait()
        results.append((ok.cpu().numpy().copy(), hd, t.aggregate_signatures().cpu().numpy().copy(), T._full(t.slashings(), n_agg * csize)[1],
                        t.discounted() if discount else None))

    n = len(epochs)
    for k, e in enumerate(epochs):
        d = [torch.as_tensor(e[x], device=dev) for x in ("sigs", "bits", "msgs", "tgt", "blk")]
        src = torch.as_tensor(e["src"], device=dev)
        kw = dict(source_epoch=src, current_epoch=T.CUR0 + k)
        keep.append((d, src))
        if mode in ("pipelined_host", "sync_host"):
            h = [x.cpu().pin_memory() for x in d]
            kw["source_epoch"] = src.cpu().pin_memory()
            keep.append((h, kw["source_epoch"]))
            if mode == "sync_host":
                ok, hd = ep.process_epoch_host(*h, **kw)
                results.append((ok.numpy().copy(), hd, ep.d_agg_sig[0].cpu().numpy().copy(), T._full(ep.slashings(), n_agg * csize)[1],
                                ep.discounted() if discount else None))
            else:
                t = ep.submit_host(*h, last=(k == n - 1), **kw)
                if t is not None:
                    collect(t)
        elif mode == "sync":
            ok, hd = ep.process_epoch_dev(*d, **kw)
            torch.cuda.synchronize()
            results.append((ok.cpu().numpy().copy(), int(hd.item()), ep.d_agg_sig[0].cpu().numpy().copy(), T._full(ep.slashings(), n_agg * csize)[1],
                            ep.discounted() if discount else None))
        else:
            t = ep.submit_dev(*d, last=(k % 3 == 2), **kw)
            if t is not None:
                collect(t)
    if mode.startswith("pipelined"):
        for t in ep.drain():
            collect(t)
    assert len(results) == n
    torch.cuda.synchronize()
    equiv = ep.equivocating()
    e_, b_, h_ = eng.latest_messages_read()
    assert eng.guard_flags() == 0
    return results, (equiv, e_, b_, h_)


def _six_epochs(mode, depth, discount, pre_marked=(), n_epochs=T.N_EPOCHS):
    members, off, tree, eff = T._world()
    eng = T._engine(tree, eff)
    epochs = T._inputs(eng, members, off)[:n_epochs]
    if pre_marked:
        eng.on_attester_slashing(sorted(pre_marked), sorted(pre_marked))
    try:
        return _run(eng, epochs, members, off, T.N_BLK, mode, depth, 16, discount)
    finally:
        eng.close()


def _check_against_oracle(run, want, final_want):
    results, final = run
    for k, ((ok, head, agg, kind, new), (w_head, w_new)) in enumerate(zip(results, want)):
        assert head == w_head, (k, head, w_head)
        assert new.tolist() == w_new.tolist(), (k, new, w_new)
    equiv, e_, b_, h_ = final
    w_equiv, w_e, w_b, w_h = final_want
    assert np.array_equal(equiv != 0, w_equiv != 0)
    assert np.array_equal(h_, w_h) and np.array_equal(e_, w_e) and np.array_equal(b_, w_b)


@pytest.mark.parametrize("mode,depth", [("sync", 3), ("sync_host", 3), ("pipelined", 2), ("pipelined", 3), ("pipelined", 4), ("pipelined_host", 3)])
def test_discount_equals_sequential_oracle(mode, depth):
    members, off, tree, eff = T._world()
    on = _six_epochs(mode, depth, True)
    off_run = _six_epochs(mode, depth, False)
    epochs = T._CACHE["inputs"]
    want, final_want = _oracle(epochs, members, off, tree, eff, T.N_VAL, 16)
    for k in range(T.N_EPOCHS):
        ok, _, agg, kind, _ = on[0][k]
        ok0, _, agg0, kind0, _ = off_run[0][k]
        assert np.array_equal(ok, ok0) and np.array_equal(ok, epochs[k]["ok"]) and np.array_equal(agg, agg0), k
        assert np.array_equal(kind, kind0), k                  # the slasher's findings do not depend on the discount
    # the planted double vote of epoch 2 is discounted (its committee), then the two surrounding aggregates of epoch 3
    assert [len(w[1]) for w in want] == [0, 0, 4, 8, 0, 0]
    _check_against_oracle(on, want, final_want)
    assert not off_run[1][0].any()                      # discounting off: nothing is marked


def test_discount_without_offence_changes_nothing():
    """epochs 0 and 1 of the world hold no offence: with discounting on every output equals a run with it off"""
    on = _six_epochs("pipelined", 3, True, n_epochs=2)
    off_run = _six_epochs("pipelined", 3, False, n_epochs=2)
    for a, b in zip(on[0], off_run[0]):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
        assert a[4].size == 0
    for x, y in zip(on[1], off_run[1]):
        assert np.array_equal(x, y)


def test_marked_before_the_run_are_not_reported_again():
    """two of the four double voters of epoch 2 were marked through on_attester_slashing before epoch 0: they never move their latest
    message, and only the other two are reported as newly discounted"""
    members, off, tree, eff = T._world()
    committee = [int(v) for v in members[off[1]:off[2]]]
    pre = sorted(committee[:2])
    run = _six_epochs("pipelined", 3, True, pre_marked=pre)
    want, final_want = _oracle(T._CACHE["inputs"], members, off, tree, eff, T.N_VAL, 16, pre_marked=pre)
    assert want[2][1].tolist() == sorted(committee[2:])
    _check_against_oracle(run, want, final_want)


# ------------------------------------------------------------------------------------------ a balancing pattern the discount defeats
def _balancing(eng, csize=4, n_agg=16):
    """blocks 0 <- A = 1, 0 <- B = 2.  Committee X (aggregate 0, heavy) votes A in epoch 0 with target CUR0; in epoch 1 it signs B with
    the same target (a double vote); in epoch 2 it votes A again.  Aggregates 1..7 vote A, 8..15 vote B throughout.  Balances: X 100 per
    member, everyone else 32, so A = 896 + 400 against B = 1024: with X counted A leads, without it B does."""
    n_val = n_agg * csize
    members = np.arange(n_val, dtype=np.uint32)
    off = (np.arange(n_agg + 1) * csize).astype(np.uint32)
    eff = np.full(n_val, 32, dtype=np.uint64)
    eff[:csize] = 100
    tree = (np.array([0, 0, 0], dtype=np.uint32), np.array([0, 1, 1], dtype=np.uint64),
            np.stack([np.full(32, 0x10, np.uint8), np.full(32, 0x20, np.uint8), np.full(32, 0x30, np.uint8)]), np.ones(3, dtype=np.uint8))
    epochs = []
    for k in range(3):
        cur = T.CUR0 + k
        src, tgt = np.full(n_agg, cur - 1, dtype=np.int64), np.full(n_agg, cur, dtype=np.int64)
        blk = np.where(np.arange(n_agg) < 8, 1, 2).astype(np.int32)
        tags = [b"bal/epoch%d/agg%d" % (k, a) for a in range(n_agg)]
        if k == 1:
            src[0], tgt[0], blk[0], tags[0] = T.CUR0 - 1, T.CUR0, 2, b"bal/X/B"
        msgs = np.frombuffer(b"".join(T._h(t) for t in tags), dtype=np.uint8).reshape(n_agg, 32).copy()
        bits = np.full((n_agg, 1), (1 << csize) - 1, dtype=np.uint8)
        sigs = eng.sign([scenarios.secret_key(int(v)) for v in members], np.repeat(np.arange(n_agg, dtype=np.uint32), csize), msgs)
        epochs.append(dict(sigs=sigs, bits=bits, msgs=msgs, src=src, tgt=tgt, blk=blk, ok=np.ones(n_agg, dtype=np.uint8)))
    return members, off, eff, tree, epochs


@pytest.mark.parametrize("mode,depth", [("sync", 3), ("pipelined", 2), ("pipelined", 3)])
def test_balancing_pattern_head_moves_only_with_discounting(mode, depth):
    from pos_evolution_b200.engine import Engine
    heads = {}
    for discount in (False, True):
        eng = Engine(0)
        members, off, eff, tree, epochs = _balancing(eng)
        eng.registry_load(eng.sk_to_pk([scenarios.secret_key(v) for v in range(len(members))]), eff)
        eng.tree_load(*tree)
        eng.latest_messages_reset()
        results, final = _run(eng, epochs, members, off, 3, mode, depth, 16, discount)
        eng.close()
        heads[discount] = [r[1] for r in results]
        assert all(r[0].all() for r in results)
        if discount:
            want, final_want = _oracle(epochs, members, off, tree, eff, len(members), 16)
            assert [w[0] for w in want] == heads[True]
            assert want[1][1].tolist() == [0, 1, 2, 3]
            _check_against_oracle((results, final), want, final_want)
    assert heads[False] == [1, 1, 1]                   # X's weight keeps A ahead
    assert heads[True] == [1, 1, 2]                    # X, caught in epoch 1, no longer counts from epoch 2: B


# ------------------------------------------------------------------------------------------ range form and error contract
@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def test_range_split_of_the_golden_streams_marks_the_union(eng):
    with open(os.path.join(HERE, "golden", "literal_slashing.json")) as f:
        golden = json.load(f)
    n, H = golden["n_validators"], golden["history_epochs"]
    eng.registry_load(eng.sk_to_pk([scenarios.secret_key(v) for v in range(n)]), np.full(n, 32, dtype=np.uint64))
    cuts = [0, n // 3, 2 * n // 3, n]
    for stream in golden["streams"]:
        batches = SO.golden_batches(stream)
        marks = {}
        for v0, v1 in [(0, n)] + list(zip(cuts[:-1], cuts[1:])):
            eng.latest_messages_reset()
            eng.slasher_init(n, H, 64, 0, v_begin=v0, v_end=v1)
            total_new = 0
            for cur, aggs in batches:
                eng.slasher_advance(cur)
                members = SO.batch(aggs)[0]
                kind = eng.slasher_update(*SO.batch(aggs))[1]
                new, n_new = eng.slasher_discount(members, kind)
                assert int(new.sum()) == n_new
                assert len(set(members[new != 0].tolist())) == n_new               # one slot per newly marked validator
                total_new += n_new
            marks[(v0, v1)] = eng.equivocating()
            assert int((marks[(v0, v1)] != 0).sum()) == total_new
            assert not marks[(v0, v1)][:v0].any() and not marks[(v0, v1)][v1:].any()
            assert eng.guard_flags() == 0
        union = np.zeros(n, dtype=np.uint8)
        for rng, m in marks.items():
            if rng != (0, n):
                union |= m
        assert np.array_equal(union != 0, marks[(0, n)] != 0)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def test_discount_marks_once_and_error_contract():
    from pos_evolution_b200._lib import B2_EINVAL
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    lib = e.lib
    members, kind = np.array([5, 5, 7, 9, 5, 6], dtype=np.uint32), np.array([1, 2, 0, 4, 1, 0], dtype=np.uint8)
    new, cnt = np.zeros(6, dtype=np.uint8), ctypes.c_uint32(0)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    d_m, d_k = torch.from_numpy(members.view(np.int32)).cuda(), torch.from_numpy(kind).cuda()
    d_new, d_cnt = torch.zeros(6, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    dev_args = (d_m.data_ptr(), d_k.data_ptr(), 6, d_new.data_ptr(), d_cnt.data_ptr(), stream)
    # no registry, then no slasher
    assert lib.b2_slasher_discount(e.h, _p(members), _p(kind), 6, _p(new), ctypes.byref(cnt)) == B2_EINVAL
    assert lib.b2_slasher_discount_dev(e.h, *dev_args) == B2_EINVAL
    assert lib.b2_equivocating_read(e.h, _p(new), 6) == B2_EINVAL
    n = 16
    e.registry_load(e.sk_to_pk([scenarios.secret_key(v) for v in range(n)]), np.full(n, 32, dtype=np.uint64))
    e.on_attester_slashing([9], [9])
    before = e.equivocating()
    assert before.tolist() == [1 if v == 9 else 0 for v in range(n)]
    assert lib.b2_slasher_discount(e.h, _p(members), _p(kind), 6, _p(new), ctypes.byref(cnt)) == B2_EINVAL
    assert lib.b2_slasher_discount_dev(e.h, *dev_args) == B2_EINVAL
    e.slasher_init(n, 8, 8, 0)
    # bad arguments
    assert lib.b2_slasher_discount(e.h, None, _p(kind), 6, _p(new), ctypes.byref(cnt)) == B2_EINVAL
    assert lib.b2_slasher_discount(e.h, _p(members), _p(kind), 0, _p(new), ctypes.byref(cnt)) == B2_EINVAL
    assert lib.b2_slasher_discount(e.h, _p(members), _p(kind), 6, None, ctypes.byref(cnt)) == B2_EINVAL
    assert lib.b2_slasher_discount_dev(e.h, d_m.data_ptr(), d_k.data_ptr(), 6, d_new.data_ptr(), None, stream) == B2_EINVAL
    assert lib.b2_equivocating_read(e.h, _p(np.zeros(n + 1, np.uint8)), n + 1) == B2_EINVAL
    d_tab = torch.ones(n, dtype=torch.uint8, device="cuda")
    for v0, v1 in ((3, 3), (4, 3), (0, n + 1), (n, n + 1)):
        assert lib.b2_equivocating_merge_dev(e.h, v0, v1, d_tab.data_ptr(), stream) == B2_EINVAL
        assert lib.b2_equivocating_slice_dev(e.h, v0, v1, d_tab.data_ptr(), stream) == B2_EINVAL
    assert lib.b2_equivocating_merge_dev(e.h, 0, 4, None, stream) == B2_EINVAL
    torch.cuda.synchronize()
    assert np.array_equal(e.equivocating(), before)       # nothing changed
    # 5 is flagged in three slots and reported once; 9 was marked before; 7 and 6 are not flagged
    new, cnt = e.slasher_discount(members, kind)
    assert new.tolist() == [1, 0, 0, 0, 0, 0] and cnt == 1
    assert np.nonzero(e.equivocating())[0].tolist() == [5, 9]
    new, cnt = e.slasher_discount(members, kind)
    assert not new.any() and cnt == 0
    # the device form, on a range slasher [4, 8): 9 and 12 lie outside it, so a stray kind byte marks nothing there
    e.slasher_init(n, 8, 8, 0, v_begin=4, v_end=8)
    d_m2 = torch.tensor([6, 12, 7, 4, 6], dtype=torch.int32, device="cuda")
    d_k2 = torch.tensor([1, 1, 0, 2, 4], dtype=torch.uint8, device="cuda")
    d_new2 = torch.full((5,), 7, dtype=torch.uint8, device="cuda")
    e.slasher_discount_dev(d_m2, d_k2, d_new2, d_cnt)
    torch.cuda.synchronize()
    assert d_new2.cpu().tolist() == [1, 0, 0, 1, 0] and int(d_cnt.item()) == 2
    assert np.nonzero(e.equivocating())[0].tolist() == [4, 5, 6, 9]
    # slice and merge
    d_slice = torch.zeros(8, dtype=torch.uint8, device="cuda")
    e.equivocating_slice_dev(2, 10, d_slice)
    torch.cuda.synchronize()
    assert d_slice.cpu().tolist() == [0, 0, 1, 1, 1, 0, 0, 1]
    e.equivocating_merge_dev(12, 16, torch.tensor([0, 1, 0, 1], dtype=torch.uint8, device="cuda"))
    assert np.nonzero(e.equivocating())[0].tolist() == [4, 5, 6, 9, 13, 15]
    assert e.guard_flags() == 0
    e.close()
