"""The slasher inside the epoch pipeline (EpochProcessor.enable_slasher) on the small world of test_gpu_epoch.py: 64 validators,
16 aggregates of 4, real signatures (bls.Sign on the GPU), six epochs with planted offences.  Every epoch's status, kind and conflict
targets must equal, byte for byte, the same batches fed through the standalone Engine.slasher_update with accept = the expected
verdicts, and the brute force of tests/slasher_oracle.py; verdicts, aggregate signatures and heads must equal a run with the slasher
off.  Also: the range form of the history (b2_slasher_init_range) over a 3-way split of the golden streams, the asynchronous window
move, and the error contract."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import scenarios
import slasher_oracle as SO
from oracle import bls_sig as B

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
N_VAL, CSIZE, N_AGG, N_BLK, N_EPOCHS = 64, 4, 16, 40, 6
CUR0 = 2                       # epoch k is processed at current epoch CUR0 + k; its honest votes are (CUR0 + k - 1, CUR0 + k)
REJECTED = (3, 7, 9)           # as in test_gpu_epoch.py: a foreign signature (3, 7), bits that do not match the signers (9)


def _h(tag):
    return hashlib.sha256(tag).digest()


def _world(n_val=N_VAL):
    """n_val >= N_VAL: the registry's size; validators N_VAL.. are in no committee (32 ETH each), so they change no vote, verdict or
    finding, only the registry's validator ranges"""
    rng = np.random.default_rng(21)
    members = rng.permutation(N_VAL).astype(np.uint32)
    off = (np.arange(N_AGG + 1) * CSIZE).astype(np.uint32)
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 5)
    eff = (rng.integers(16, 33, size=N_VAL).astype(np.uint64)) * np.uint64(10**9)
    eff = np.concatenate([eff, np.full(n_val - N_VAL, 32 * 10**9, dtype=np.uint64)])
    return members, off, (parent, slot, roots, leaf_viable), eff


def _plan(k):
    """(source, target, message tag, bad signature) of every aggregate of epoch k; the planted offences:
      k=2 agg 1   (k, k+1) another message: a double vote of its whole committee (its honest vote of epoch 1 had that target);
      k=3 agg 2   (k-1, k+2): surrounds its (k, k+1) vote of the epoch before;
      k=3 agg 6   (0, k+2): surrounds (1, 2), (2, 3) and (3, 4);
      k=3 agg 10  (0, k+2) with a foreign signature: rejected, so neither recorded nor flagged;
      k=4 agg 6   its epoch-2 vote (3, 4) again, same message: surrounded by its (0, 5), and no double vote;
      k=4 agg 10  its epoch-2 vote again: an identical re-vote (flagged only if the rejected (0, 5) had been recorded);
      k=5 agg 8   its epoch-4 vote again: an identical re-vote."""
    cur = CUR0 + k
    plan = [[cur - 1, cur, b"epoch%d/agg%d" % (k, a), a in (3, 7)] for a in range(N_AGG)]
    if k == 2:
        plan[1] = [cur - 2, cur - 1, b"other%d/agg1" % k, False]
    if k == 3:
        plan[2] = [cur - 3, cur, plan[2][2], False]
        plan[6] = [0, cur, plan[6][2], False]
        plan[10] = [0, cur, plan[10][2], True]
    if k == 4:
        plan[6] = [3, 4, b"epoch2/agg6", False]
        plan[10] = [3, 4, b"epoch2/agg10", False]
    if k == 5:
        plan[8] = [5, 6, b"epoch4/agg8", False]
    return plan


EXPECTED_FLAGGED = {2: 4, 3: 8, 4: 4}


_CACHE = {}


def _inputs(eng, members, off):
    """per epoch: sigs u8[64, 96], bits, msgs, source, target, block, expected verdicts -- signed once on the GPU (bls.Sign)"""
    if "inputs" in _CACHE:
        return _CACHE["inputs"]
    out = []
    for k in range(N_EPOCHS):
        plan = _plan(k)
        msgs = np.frombuffer(b"".join(_h(p[2]) for p in plan), dtype=np.uint8).reshape(N_AGG, 32).copy()
        bits = np.full((N_AGG, 1), 0x0F, dtype=np.uint8)
        bits[5, 0], bits[9, 0] = 0x0B, 0x07
        signers = [int(v) for v in members]
        msg_idx = np.repeat(np.arange(N_AGG, dtype=np.uint32), CSIZE)
        sigs = eng.sign([scenarios.secret_key(v) for v in signers], msg_idx, msgs)
        for a, p in enumerate(plan):
            if p[3]:                                            # one member's signature by another validator: the aggregate fails
                j = int(off[a]) + 1
                sigs[j] = eng.sign([scenarios.secret_key((signers[j] + 1) % N_VAL)], [0], msgs[a:a + 1])[0]
        sigs[int(off[5]) + 2] = np.frombuffer(bytes([0xC0]) + bytes(95), dtype=np.uint8)   # the non-signer of aggregate 5: the identity
        src = np.array([p[0] for p in plan], dtype=np.int64)
        tgt = np.array([p[1] for p in plan], dtype=np.int64)
        blk = ((np.arange(N_AGG) * 7 + 3 * k) % N_BLK).astype(np.int32)
        ok = np.array([0 if (a in (3, 7, 9) or plan[a][3]) else 1 for a in range(N_AGG)], dtype=np.uint8)
        out.append(dict(sigs=sigs, bits=bits, msgs=msgs, src=src, tgt=tgt, blk=blk, ok=ok))
    # the verdicts the construction implies, checked against the oracle's FastAggregateVerify where an offence was planted
    pks = scenarios.pubkeys(N_VAL)
    for k, a in ((2, 1), (3, 2), (3, 10), (4, 6)):
        e = out[k]
        seg = [bytes(s) for s in e["sigs"][off[a]:off[a + 1]]]
        sel = [int(members[off[a] + j]) for j in range(CSIZE) if (e["bits"][a, 0] >> j) & 1]
        assert int(B.FastAggregateVerify([pks[v] for v in sel], bytes(e["msgs"][a]), B.Aggregate(seg))) == e["ok"][a], (k, a)
    _CACHE["inputs"] = out
    return out


def _engine(tree, eff, device=0):
    from pos_evolution_b200.engine import Engine
    parent, slot, roots, leaf_viable = tree
    eng = Engine(device)
    pk = eng.sk_to_pk([scenarios.secret_key(v) for v in range(len(eff))])
    eng.registry_load(pk, eff)
    eng.tree_load(parent, slot, roots, leaf_viable)
    eng.latest_messages_reset()
    return eng


def _full(sl, total):
    """a Slashings report -> (status, kind u8[total], conflict u32[total, 2], n_flagged) in the layout of Engine.slasher_update"""
    kind = np.zeros(total, dtype=np.uint8)
    conflict = np.full((total, 2), SO.NO_TARGET, dtype=np.uint32)
    slots = (np.asarray(sl.aggregate) * CSIZE + np.asarray(sl.position)).astype(np.int64)
    kind[slots] = sl.kind
    conflict[slots, 0], conflict[slots, 1] = sl.surrounded_target, sl.surrounding_target
    return sl.status, kind, conflict, len(slots)


def _run(mode, depth, H, slasher, n_val=N_VAL):
    """the six epochs through EpochProcessor in `mode`, on a registry of n_val; -> per epoch (verdicts, head, aggregate signatures,
    Slashings or None)"""
    from pos_evolution_b200.epoch import EpochProcessor
    members, off, tree, eff = _world(n_val)
    eng = _engine(tree, eff)
    epochs = _inputs(eng, members, off)
    dev = torch.device("cuda", 0)
    ep = EpochProcessor(eng, N_AGG, N_AGG * CSIZE, 1, N_BLK, device=dev, depth=depth, tail_form="thread")
    ep.set_committees(members, off)
    if slasher:
        ep.enable_slasher(H, current_epoch=CUR0)
    results, keep = [], []

    def collect(t):
        ok, hd = t.wait()
        results.append((ok.cpu().numpy().copy(), hd, t.aggregate_signatures().cpu().numpy().copy(), t.slashings() if slasher else None))

    for k, e in enumerate(epochs):
        d = [torch.as_tensor(e["sigs"], device=dev), torch.as_tensor(e["bits"], device=dev), torch.as_tensor(e["msgs"], device=dev),
             torch.as_tensor(e["tgt"], device=dev), torch.as_tensor(e["blk"], device=dev)]
        src = torch.as_tensor(e["src"], device=dev)
        kw = dict(source_epoch=src, current_epoch=CUR0 + k) if slasher else {}
        keep.append((d, src))
        if mode in ("pipelined_host", "sync_host"):
            h = [x.cpu().pin_memory() for x in d]
            hs = src.cpu().pin_memory()
            keep.append((h, hs))
            if slasher:
                kw["source_epoch"] = hs
            if mode == "sync_host":
                ok, hd = ep.process_epoch_host(*h, **kw)
                results.append((ok.numpy().copy(), hd, ep.d_agg_sig[0].cpu().numpy().copy(), ep.slashings() if slasher else None))
            else:
                t = ep.submit_host(*h, last=(k == N_EPOCHS - 1), **kw)
                if t is not None:
                    collect(t)
        elif mode == "sync":
            ok, hd = ep.process_epoch_dev(*d, **kw)
            torch.cuda.synchronize()
            results.append((ok.cpu().numpy().copy(), int(hd.item()), ep.d_agg_sig[0].cpu().numpy().copy(), ep.slashings() if slasher else None))
        else:
            t = ep.submit_dev(*d, last=(k % 3 == 2), **kw)
            if t is not None:
                collect(t)
    if mode.startswith("pipelined"):
        for t in ep.drain():
            collect(t)
    assert len(results) == N_EPOCHS
    assert eng.guard_flags() == 0
    eng.close()
    return results


@pytest.mark.parametrize("mode,depth,H", [("pipelined", 2, 16), ("pipelined", 3, 16), ("pipelined", 4, 16), ("sync", 3, 16), ("sync_host", 3, 16),
                                          ("pipelined_host", 3, 16), ("pipelined", 3, 4), ("pipelined_host", 4, 4)])
def test_epoch_slasher_equals_standalone_and_brute_force(mode, depth, H):
    """H = 4: the window moves across ring wraps through slasher_advance_dev (one column per epoch, on the fork-choice stream), the
    standalone run through the synchronous slasher_advance; the long spans of epoch 3 start below the window there (SOURCE_EXPIRED)."""
    from pos_evolution_b200.engine import Engine
    members, off, tree, eff = _world()
    on = _run(mode, depth, H, True)
    off_run = _run(mode, depth, H, False)
    ref = Engine(0)
    K = 2 * N_AGG
    ref.slasher_init(N_VAL, H, K, CUR0)
    bs = SO.BruteSlasher(N_VAL, H, K, CUR0)
    epochs = _CACHE["inputs"]
    for k, e in enumerate(epochs):
        ok, head, agg, sl = on[k]
        ok0, head0, agg0, _ = off_run[k]
        assert np.array_equal(ok, e["ok"]) and np.array_equal(ok, ok0), k
        assert head == head0 and np.array_equal(agg, agg0), k
        ref.slasher_advance(CUR0 + k)
        bs.advance(CUR0 + k)
        args = (members, off, e["bits"], e["src"].astype(np.uint64), e["tgt"].astype(np.uint64), e["msgs"])
        want = ref.slasher_update(*args, e["ok"])
        brute = bs.update(*args, e["ok"])
        got = _full(sl, N_AGG * CSIZE)
        for g, w, b, what in zip(got, want, brute, ("status", "kind", "conflict", "n_flagged")):
            assert np.array_equal(g, w), (k, what, g, w)
            assert np.array_equal(w, b), (k, what, w, b)
        assert np.array_equal(sl.validator, members[np.asarray(sl.aggregate) * CSIZE + np.asarray(sl.position)])
        if H == 16:
            assert got[3] == EXPECTED_FLAGGED.get(k, 0), (k, got[3])
            assert got[0][10] == (SO.NOT_ACCEPTED if k == 3 else SO.OK)
            if k == 2:
                assert set(sl.aggregate.tolist()) == {1} and set(sl.kind.tolist()) == {SO.DOUBLE}
            if k == 3:
                assert sorted(set(zip(sl.aggregate.tolist(), sl.kind.tolist(), sl.surrounded_target.tolist()))) == [(2, SO.SURROUNDS, 4), (6, SO.SURROUNDS, 2)]
            if k == 4:
                assert set(zip(sl.aggregate.tolist(), sl.kind.tolist(), sl.surrounding_target.tolist())) == {(6, SO.SURROUNDED, 5)}
    ref.close()


# ------------------------------------------------------------------------------------------ range form and error contract
@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def test_range_split_of_the_golden_streams_equals_the_full_range(eng):
    with open(os.path.join(HERE, "golden", "literal_slashing.json")) as f:
        golden = json.load(f)
    n, H = golden["n_validators"], golden["history_epochs"]
    cuts = [0, n // 3, 2 * n // 3, n]
    for stream in golden["streams"]:
        batches = SO.golden_batches(stream)
        runs = []
        for v0, v1 in [(0, n)] + list(zip(cuts[:-1], cuts[1:])):
            eng.slasher_init(n, H, 64, 0, v_begin=v0, v_end=v1)
            outs = []
            for cur, aggs in batches:
                eng.slasher_advance(cur)
                outs.append(eng.slasher_update(*SO.batch(aggs)))
            assert eng.guard_flags() == 0                           # out-of-range members are skipped without a guard bit
            runs.append(((v0, v1), outs))
        (_, full), parts = runs[0], runs[1:]
        for i, (cur, aggs) in enumerate(batches):
            members = SO.batch(aggs)[0]
            status, kind, conflict, n_flagged = full[i]
            union_kind = np.zeros_like(kind)
            union_conflict = np.full_like(conflict, SO.NO_TARGET)
            for (v0, v1), outs in parts:
                p_status, p_kind, p_conflict, _ = outs[i]
                assert np.array_equal(p_status, status)                # per-aggregate state does not depend on the range
                outside = (members < v0) | (members >= v1)
                assert not p_kind[outside].any() and (p_conflict[outside] == SO.NO_TARGET).all()
                union_kind |= p_kind
                inside = ~outside
                union_conflict[inside] = p_conflict[inside]
            assert np.array_equal(union_kind, kind) and np.array_equal(union_conflict, conflict), i
            assert sum(outs[i][3] for _, outs in parts) == n_flagged


def test_range_device_guard_and_out_of_range_members(eng):
    """device form on a range [8, 16) of 32: an index >= 32 still sets B2_GUARD_BAD_INDEX; members outside the range are silent"""
    n = 32
    eng.slasher_init(n, 8, 8, 10, v_begin=8, v_end=16)
    members = np.array([3, 9, 20, 40, 10], dtype=np.uint32)
    off = np.array([0, 4, 5], dtype=np.uint32)
    bits = np.full((2, 1), 0xFF, dtype=np.uint8)
    src, tgt = np.array([9, 8], dtype=np.uint64), np.array([10, 10], dtype=np.uint64)
    roots = np.frombuffer(SO.root_of(1) + SO.root_of(2), dtype=np.uint8).reshape(2, 32)
    dev = [torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x.view(np.int32) if x.dtype == np.uint32 else x.copy()).cuda()
           for x in (members, off, bits, src, tgt, roots)]
    d_status = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    d_kind = torch.zeros(5, dtype=torch.uint8, device="cuda")
    d_conflict = torch.zeros((5, 2), dtype=torch.int32, device="cuda")
    d_flagged = torch.zeros(1, dtype=torch.int32, device="cuda")
    eng.guard_flags()
    eng.slasher_update_dev(*dev, None, d_status, d_kind, d_conflict, d_flagged)
    assert eng.guard_flags() == 1                                  # B2_GUARD_BAD_INDEX for 40 only
    assert d_status.cpu().tolist() == [SO.OK, SO.OK]
    assert d_kind.cpu().tolist() == [0, 0, 0, 0, 0] and int(d_flagged.item()) == 0
    status, kind, conflict, nf = eng.slasher_update(*SO.batch([([3, 9, 20, 10], 9, 10, SO.root_of(3))]))
    assert kind.tolist() == [0, SO.DOUBLE, 0, SO.DOUBLE] and nf == 2        # 3 and 20 double-voted too, but another range holds them
    assert conflict[0].tolist() == [SO.NO_TARGET, SO.NO_TARGET] and eng.guard_flags() == 0


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def test_range_and_advance_dev_error_contract(eng):
    from pos_evolution_b200._lib import B2_EINVAL, B2_ENOMEM, B2Error
    lib = eng.lib
    eng.slasher_init(16, 8, 8, 10, v_begin=4, v_end=12)
    bs = SO.BruteSlasher(16, 8, 8, 10)
    first = SO.batch([([4, 5], 8, 10, SO.root_of(1))])
    assert np.array_equal(eng.slasher_update(*first)[1], bs.update(*first)[1])
    for v0, v1 in ((5, 5), (6, 5), (0, 17), (16, 17)):
        assert lib.b2_slasher_init_range(eng.h, 16, v0, v1, 8, 8, 10) == B2_EINVAL
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.b2_slasher_advance_dev(eng.h, 9, stream) == B2_EINVAL                # backwards
    assert lib.b2_slasher_advance_dev(eng.h, 2**32 - 1, stream) == B2_EINVAL        # does not fit 32 bits
    with pytest.raises(B2Error) as e:                      # 6 * 2^24 * 65 535 bytes: refused by arithmetic before any allocation
        eng.slasher_init(1 << 24, 65535, 16, 0, v_begin=0, v_end=1 << 24)
    assert e.value.code == B2_ENOMEM
    free0 = torch.cuda.mem_get_info()[0]
    assert lib.b2_slasher_init_range(eng.h, 1 << 24, 1 << 20, 1 << 24, 65535, 16, 0) == B2_ENOMEM
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
    # the previous slasher is intact: window, tables and range
    second = SO.batch([([4, 5, 13], 9, 10, SO.root_of(2)), ([5], 7, 11, SO.root_of(3))])
    status, kind, conflict, nf = eng.slasher_update(*second)
    want = bs.update(*second)
    assert status.tolist() == [SO.OK, SO.TARGET_AHEAD] and kind.tolist() == [SO.DOUBLE, SO.DOUBLE, 0, 0]
    assert np.array_equal(kind, want[1]) and nf == 2
    eng.slasher_advance_dev(11)
    torch.cuda.synchronize()                               # the host form runs on the library's own stream
    bs.advance(11)
    third = SO.batch([([5, 6], 7, 11, SO.root_of(3))])
    got, want = eng.slasher_update(*third), bs.update(*third)
    assert got[1].tolist() == [SO.SURROUNDS, 0] and got[2][0].tolist() == [10, SO.NO_TARGET]
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_enabled_slasher_requires_source_and_current_epoch():
    from pos_evolution_b200.epoch import EpochProcessor
    members, off, tree, eff = _world()
    eng = _engine(tree, eff)
    dev = torch.device("cuda", 0)
    ep = EpochProcessor(eng, N_AGG, N_AGG * CSIZE, 1, N_BLK, device=dev, depth=3)
    ep.set_committees(members, off)
    ep.enable_slasher(8, current_epoch=CUR0)
    assert ep.sl_range == (0, N_VAL) and ep.slots[0].sl_kind.numel() == N_AGG * CSIZE
    e = _inputs(eng, members, off)[0]
    d = [torch.as_tensor(e[x], device=dev) for x in ("sigs", "bits", "msgs", "tgt", "blk")]
    src = torch.as_tensor(e["src"], device=dev)
    h = [x.cpu().pin_memory() for x in d]
    for call in (lambda: ep.submit_dev(*d), lambda: ep.submit_dev(*d, source_epoch=src), lambda: ep.submit_dev(*d, current_epoch=CUR0),
                 lambda: ep.process_epoch_dev(*d, current_epoch=CUR0), lambda: ep.submit_host(*h, source_epoch=src.cpu()),
                 lambda: ep.process_epoch_host(*h), lambda: ep.submit_dev(*d, source_epoch=src, current_epoch=CUR0 - 1)):
        with pytest.raises(AssertionError):
            call()
    assert ep.k == 0 and not ep._inflight                  # nothing was enqueued
    ok, hd = ep.process_epoch_dev(*d, source_epoch=src, current_epoch=CUR0)
    assert ep.slashings().status.tolist() == [SO.NOT_ACCEPTED if a in REJECTED else SO.OK for a in range(N_AGG)]
    eng.close()
