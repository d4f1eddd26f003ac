"""GPU parity of the SingleAttestation intake (Engine.single_attestation_intake / _dev, EpochProcessor.intake_single_dev): both forms
against tests/single_intake_oracle.py on every status 0-13 at the minimal and mainnet committee counts, random epochs, committee sizes
1..2 048; the fingerprint-collision and near-miss-root epochs of test_gpu_intake_keys written as SingleAttestations; equivalence with the
phase 0 intake on the same votes; the end-to-end vote form through submit_dev; the host form's refusals and the device guards; a full
2^20-validator epoch."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch

import intake_keys as K
import intake_oracle as IO
import single_intake_oracle as SO
import test_gpu_intake as T
import test_gpu_intake_keys as KT
import test_oracle_single_intake as OS
from oracle.spec import Spec

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
DOMAIN = T.DOMAIN
EPOCH = OS.EPOCH
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _single_dev(eng, wires, subnets, members, off, epoch, cur, mv, cps, spe, stride, woff=None):
    """Engine.single_attestation_intake_dev on device tensors; the results as numpy arrays"""
    from pos_evolution_b200.engine import IntakeResult
    wire, w_off = T._wire(wires)
    woff = w_off if woff is None else woff
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32), device=DEV)      # noqa: E731
    n_sig, n_c = int(off[-1]), len(off) - 1
    z = lambda *s, dt=torch.uint8: torch.zeros(s, dtype=dt, device=DEV)      # noqa: E731
    out = [z(len(wires), dt=torch.int32), torch.full((n_sig,), -1, dtype=torch.int32, device=DEV), z(n_c + 1, dt=torch.int32), z(n_sig, 96),
           z(mv, 128), z(mv, 32), z(mv, dt=torch.int64), z(mv, dt=torch.int64), z(mv, dt=torch.int32)]
    d_wire = torch.as_tensor(np.frombuffer(wire or bytes(1), dtype=np.uint8).copy(), device=DEV)
    eng.single_attestation_intake_dev(d_wire, t(woff), t(subnets), t(members), t(off), epoch, cur, DOMAIN, cps, spe, stride, *out)
    torch.cuda.synchronize()
    a = [x.cpu().numpy() for x in out]
    return IntakeResult(a[0], a[1].view(np.uint32), a[2].view(np.uint32), a[3], a[4], a[5], a[6].view(np.uint64), a[7].view(np.uint64),
                        a[8].view(np.uint32))


def _both(eng, wires, subnets, members, off, epoch, cur, cps, spe, stride, want, mv=None):
    """both forms against an oracle result"""
    mv = int(want.vote_off[-1]) + 3 if mv is None else mv
    got = eng.single_attestation_intake(*T._wire(wires), subnets, members, off, epoch, cur, DOMAIN, cps, spe, stride, mv)
    T._assert_equal(got, want, mv)
    T._assert_equal(_single_dev(eng, wires, subnets, members, off, epoch, cur, mv, cps, spe, stride), want, mv)
    assert eng.guard_flags() == 0


def _oracle(wires, subnets, members, off, tree, epoch, cur, cps, spe):
    blocks, ids = IO.block_store(*tree)
    return SO.single_intake_plain(wires, subnets, members, off, epoch, cur, DOMAIN, cps, spe, blocks, ids)


# ------------------------------------------------------------------------------------------ phase 0 epochs written as SingleAttestations
def to_single(w0, members, off, cps, spe, epoch):
    """a one-bit phase 0 Attestation as the SingleAttestation of the same vote: committee_index = data.index, data.index = 0, the
    attester at the bit's position"""
    w0 = bytes(w0)
    slot, index = int.from_bytes(w0[4:12], "little"), int.from_bytes(w0[12:20], "little")
    bits = w0[228:]
    p = next(8 * i + (b & -b).bit_length() - 1 for i, b in enumerate(bits) if b)
    c = (slot - epoch * spe) * cps + index
    d = w0[4:12] + bytes(8) + w0[20:132]
    return SO.encode(index, int(members[int(off[c]) + p]), d, w0[132:228])


def single_want(want0):
    """the phase 0 oracle's result as the SingleAttestation form gives it: each vote's data with data.index = 0 and its signing root"""
    import types
    d = want0.data128.copy()
    msgs = want0.msgs.copy()
    for v in range(d.shape[0]):
        if msgs[v].any():
            d[v, 8:16] = 0
            msgs[v] = np.frombuffer(Spec.compute_signing_root(IO.data_from_bytes(bytes(d[v])), DOMAIN), np.uint8)
    return types.SimpleNamespace(status=want0.status, vote=want0.vote, vote_off=want0.vote_off, sigs=want0.sigs, data128=d, msgs=msgs,
                                 source_epoch=want0.source_epoch, target_epoch=want0.target_epoch, block_idx=want0.block_idx)


# ------------------------------------------------------------------------------------------ every status, random epochs
@pytest.mark.parametrize("spe,cps,size", OS.PRESETS, ids=["minimal", "mainnet"])
def test_every_status_both_forms(eng, spe, cps, size):
    tree = OS._tree(spe)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    members, off = OS._committees(spe * cps, size)
    wires, subnets, cur = OS.every_status_case(tree, spe, cps, members, off)
    want = _oracle(wires, subnets, members, off, tree, EPOCH, cur, cps, spe)
    assert set(want.status.tolist()) == set(range(14))
    few = _oracle(wires[:3], subnets[:3], members, off, tree, EPOCH, cur, cps, spe)
    _both(eng, wires[:3], subnets[:3], members, off, EPOCH, cur, cps, spe, 1, few)
    _both(eng, wires, subnets, members, off, EPOCH, cur, cps, spe, 1, want)
    _both(eng, wires[:3], subnets[:3], members, off, EPOCH, cur, cps, spe, 1, few)      # on the scratch the full list grew


@pytest.mark.parametrize("seed", range(4))
def test_random_epochs_match_oracle(eng, seed):
    spe, cps, size = 8, 3, 9
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, 60, EPOCH * spe - 7)
    eng.tree_load(*tree, np.ones(60, np.uint8))
    members, off = OS._committees(spe * cps, size, seed=seed)
    wires, subnets = SO.random_epoch(rng, EPOCH, spe, cps, members, off, tree, len(members), corrupt=0.4, dup=0.2, heads_per_committee=3)
    cur = EPOCH * spe + 4 if seed == 3 else (EPOCH + 1) * spe + 1      # seed 3: the later slots' items are status 7
    want = _oracle(wires, subnets, members, off, tree, EPOCH, cur, cps, spe)
    assert {0, 1, 8, 13} <= set(want.status.tolist()) and (seed != 3 or 7 in want.status)
    _both(eng, wires, subnets, members, off, EPOCH, cur, cps, spe, 2, want)
    _both(eng, wires, subnets, members, off, EPOCH, cur, cps, spe, 2, want, mv=spe * cps + 2)      # fewer rows than votes


# ------------------------------------------------------------------------------------------ committee sizes, equivalence with phase 0
SIZES = [1, 2, 7, 8, 9, 31, 255, 256, 257, 1000, 2047, 2048]


@pytest.mark.parametrize("size", SIZES)
def test_committee_sizes_and_phase0_equivalence(eng, size):
    """a ragged epoch of phase 0 votes (committee c of size `size` or a neighbour) written as SingleAttestations: both forms match the
    oracle, and give the phase 0 intake's vote, vote_off, sigs, epochs and block ids on the phase 0 wires, data128 apart from bytes 8-15"""
    spe, cps = 2, 2
    rng = np.random.default_rng(size)
    tree = IO.random_tree(rng, 30, EPOCH * spe - 4)
    eng.tree_load(*tree, np.ones(30, np.uint8))
    sizes = [size, max(1, size - 1), size, min(2048, size + 1)]
    off = IO.ragged_layout(sizes)
    members = rng.permutation(int(off[-1]) + 50)[:int(off[-1])].astype(np.uint32)
    stride = 256 if size > 1024 else max(1, (size + 8) // 8)
    w0 = IO.ragged_epoch(rng, EPOCH, spe, cps, sizes, tree, distinct=3, absent=0.1, dup=0.1)
    wires = [to_single(w, members, off, cps, spe, EPOCH) for w in w0]
    subnets = SO.subnets_of(wires, cps, spe)
    cur = (EPOCH + 1) * spe
    want = _oracle(wires, subnets, members, off, tree, EPOCH, cur, cps, spe)
    _both(eng, wires, subnets, members, off, EPOCH, cur, cps, spe, stride, want)
    mv = int(want.vote_off[-1])
    p0 = eng.attestation_intake(*T._wire(w0), off, EPOCH, cur, DOMAIN, cps, spe, stride, mv)
    s1 = eng.single_attestation_intake(*T._wire(wires), subnets, members, off, EPOCH, cur, DOMAIN, cps, spe, stride, mv)
    assert np.array_equal(p0.status, s1.status)
    for f in ("vote", "vote_off", "sigs", "source_epoch", "target_epoch", "block_idx"):
        assert np.array_equal(getattr(p0, f), getattr(s1, f)), f
    diff = p0.data128 != s1.data128
    assert not diff[:, :8].any() and not diff[:, 16:].any()


# ------------------------------------------------------------------------------------------ colliding fingerprints, near-miss roots
@pytest.mark.parametrize("k", [2, 33, 257])
@pytest.mark.parametrize("size", [64, 2048])
def test_collision_sets(eng, size, k):
    """test_gpu_intake_keys' collision epochs: zeroing data.index moves every datum of a committee by the same amount, so each
    committee's data still share one fingerprint"""
    spe = cps = 2
    stride = size // 8
    tree, w0, off, _ = KT._collision_epoch(100 * k + size, size, k)
    members = np.random.default_rng(k).permutation(int(off[-1])).astype(np.uint32)
    wires = [to_single(w, members, off, cps, spe, EPOCH) for w in w0]
    for c in range(spe * cps):
        fps = {K.fingerprint(w[16:144]) for w in wires if int.from_bytes(w[0:8], "little") == c % cps
               and int.from_bytes(w[16:24], "little") == EPOCH * spe + c // cps}
        assert len(fps) == 1
    want = single_want(KT._numpy_oracle(tree, w0, off, spe, cps, stride))
    assert {0, 13} <= set(want.status.tolist())
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    _both(eng, wires, SO.subnets_of(wires, cps, spe), members, off, EPOCH, (EPOCH + 1) * spe, cps, spe, stride, want)


@pytest.mark.parametrize("form", ["loaded", "pruned"])
def test_near_miss_roots(eng, form):
    """test_gpu_intake_keys' root epochs: every tree root, its one-byte neighbours and ff..ff as head and as target"""
    rng = np.random.default_rng(len(form))
    parent, slot, roots, hubs, anchor = KT._tree_form(eng, form)
    tree = (parent, slot, roots)
    n = len(parent)
    valid_head = n - 1 if n > 1 else 0
    gone = [bytes(r) for r in KT._root_world()[2][[0, 2]]] if form == "pruned" else []
    w0, off, _ = KT._intake_roots(rng, tree, anchor, valid_head, gone)
    spe, cps = KT.SPE_C, KT.CPS_C
    members = rng.permutation(int(off[-1])).astype(np.uint32)
    wires = [to_single(w, members, off, cps, spe, EPOCH) for w in w0]
    want = single_want(KT._numpy_oracle(tree, w0, off, spe, cps, KT.STRIDE_C))
    assert {0, 9, 10, 12} <= set(want.status.tolist())
    _both(eng, wires, SO.subnets_of(wires, cps, spe), members, off, EPOCH, (EPOCH + 1) * spe, cps, spe, KT.STRIDE_C, want)


# ------------------------------------------------------------------------------------------ end to end through the vote form
@pytest.mark.parametrize("mode", ["sync", "pipelined", "slasher"])
def test_end_to_end_matches_oracle(eng, mode):
    """test_gpu_intake's end-to-end epochs (one committee per slot, so the phase 0 data already has data.index = 0 and the same signing
    root) written as SingleAttestations, through intake_single_dev and the vote form: the verdicts, heads, aggregates and bit rows the
    oracle computes for the phase 0 wires"""
    from pos_evolution_b200.epoch import EpochProcessor
    spe, cps, csize = T.SPE, T.E2E_CPS, T.E2E_CSIZE
    n_c = spe * cps
    tree = T._tree(seed=3, n_blocks=40, first_slot=EPOCH * spe - 5)
    n_val = n_c * csize
    import scenarios
    pks = scenarios.pubkeys(n_val)
    members = np.random.default_rng(9).permutation(n_val).astype(np.uint32)
    off = T._layout(csize, n_c)
    eff = np.full(n_val, 32 * 10**9, np.uint64)
    epochs = [T._e2e_epoch(eng, k, tree, members, off) for k in range(3)]
    want = T._e2e_expected(pks, members, off, tree, eff, epochs)
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    eng.latest_messages_reset()
    ep = EpochProcessor(eng, n_c, n_val, 1, len(tree[0]), device=DEV, depth=3, max_votes=3 * n_c)
    ep.set_committees(members, off)
    if mode == "slasher":
        ep.enable_slasher(8, current_epoch=EPOCH, discount=True)
    side = torch.cuda.Stream()
    got, keep = [], []

    def collect(t):
        ok, hd = t.wait()
        got.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().copy(), t.aggregation_bits().cpu().numpy().copy()))
    for k, (w0, e) in enumerate(epochs):
        wires = [to_single(w, members, off, cps, spe, e) for w in w0]
        wire, woff = T._wire(wires)
        subnets = SO.subnets_of(wires, cps, spe)
        with torch.cuda.stream(side):
            r = ep.intake_single_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV),
                                     torch.as_tensor(subnets.view(np.int32), device=DEV), e, (e + 1) * spe, DOMAIN, cps, spe)
        assert np.array_equal(r.status.cpu().numpy(), want[k][0].status)
        assert np.array_equal(r.vote_off, want[k][0].vote_off)
        keep.append(r)
        sl = dict(source_epoch=r.source_epoch, current_epoch=e) if mode == "slasher" else {}
        if mode == "sync":
            ok, hd = ep.process_epoch_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, votes=(r.vote, r.vote_off))
            s = ep.slots[0]
            n = int(r.vote_off[-1])
            got.append((ok.cpu().numpy().tolist(), int(hd.item()), s.agg_sig[:n].cpu().numpy().copy(), s.v_aggbits[:n].cpu().numpy().copy()))
        else:
            t = ep.submit_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, last=(k == len(epochs) - 1), votes=(r.vote, r.vote_off), **sl)
            if t is not None:
                collect(t)
    if mode != "sync":
        for t in ep.drain():
            collect(t)
    assert eng.guard_flags() == 0
    for k, (r, aggs, oks, rows, head) in enumerate(want):
        g_ok, g_head, g_agg, g_rows = got[k]
        assert g_ok == oks, k
        assert g_head == head, k
        assert [bytes(a) for a in g_agg] == aggs, k
        assert [int(x[0]) for x in g_rows] == rows, k
    assert 0 in want[0][2] and 1 in want[0][2]


def test_processor_refusals(eng):
    from pos_evolution_b200.epoch import EpochProcessor
    tree = OS._tree(8)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    members, off = OS._committees(16, 4)
    import scenarios
    eng.registry_load(np.frombuffer(b"".join(scenarios.pubkeys(64)), dtype=np.uint8), np.full(64, 32 * 10**9, np.uint64))
    ep = EpochProcessor(eng, 16, 64, 1, len(tree[0]), device=DEV)
    ep.set_committees(members, off)
    d = torch.zeros(240, dtype=torch.uint8, device=DEV)
    woff = torch.tensor([0, 240], dtype=torch.int32, device=DEV)
    sub = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="max_votes"):
        ep.intake_single_dev(d, woff, sub, EPOCH, EPOCH * 8 + 9, DOMAIN, 2, 8)
    ep = EpochProcessor(eng, 16, 64, 1, len(tree[0]), device=DEV, max_votes=32)
    ep.set_committees(members, off)
    with pytest.raises(ValueError, match="n_agg"):
        ep.intake_single_dev(d, woff, sub, EPOCH, EPOCH * 8 + 9, DOMAIN, 4, 8)
    r = ep.intake_single_dev(d, woff, sub, EPOCH, EPOCH * 8 + 9, DOMAIN, 2, 8)
    assert r.status.cpu().tolist() == [4]                  # zero bytes: slot 0 lies outside epoch 3
    assert r.vote_off.tolist() == list(range(17))


# ------------------------------------------------------------------------------------------ host refusals, device guards
def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _raw_call(e, wire, woff, subnets, members, off, epoch, cur, cps, spe, n_c=None, subnet_count=64, mv=16):
    n_att, n_sig = len(woff) - 1, int(off[-1])
    n_c = len(off) - 1 if n_c is None else n_c
    outs = [np.full(sz, SENTINEL, np.uint8) for sz in (4 * n_att, 4 * n_sig, 4 * (len(off)), 96 * n_sig, 128 * mv, 32 * mv, 8 * mv, 8 * mv, 4 * mv)]
    w = np.frombuffer(wire, np.uint8)
    rc = e.lib.b2_single_attestation_intake(e.h, _p(w), len(wire), _p(np.asarray(woff, np.uint32)), n_att,
                                            None if subnets is None else _p(np.asarray(subnets, np.uint32)), subnet_count,
                                            None if members is None else _p(np.asarray(members, np.uint32)), _p(np.asarray(off, np.uint32)),
                                            n_c, cps, spe, 1, epoch, cur, _p(np.frombuffer(DOMAIN, np.uint8)), mv, *[_p(o) for o in outs])
    return rc, outs


def test_rejected_host_calls_change_nothing(eng):
    from pos_evolution_b200 import _lib
    from pos_evolution_b200.engine import Engine
    spe, cps, size = 8, 4, 5
    tree = OS._tree(spe)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    members, off = OS._committees(spe * cps, size)
    wires, subnets, cur = OS.every_status_case(tree, spe, cps, members, off)
    wire, woff = T._wire(wires)
    weights, head = eng.get_weights(), eng.get_head(0)
    rc, _ = _raw_call(eng, wire, woff, subnets, members, off, EPOCH, cur, cps, spe)
    assert rc == 0
    bad_woff = woff.copy()
    bad_woff[3], bad_woff[4] = bad_woff[4], bad_woff[3]
    past = woff.copy()
    past[-1] += 1
    big = off.copy()
    big[1] = big[0] + 9                                     # a committee wider than 8 * bits_stride
    cases = [dict(woff=bad_woff), dict(woff=past), dict(n_c=spe * cps - 1), dict(epoch=EPOCH + 1), dict(epoch=EPOCH - 2),
             dict(cur=cur + 100), dict(subnets=None), dict(members=None), dict(subnet_count=0), dict(off=big)]
    for kw in cases:
        a = dict(woff=woff, subnets=subnets, members=members, off=off, epoch=EPOCH, cur=cur, n_c=None, subnet_count=64)
        a.update(kw)
        rc, outs = _raw_call(eng, wire, a["woff"], a["subnets"], a["members"], a["off"], a["epoch"], a["cur"], cps, spe, n_c=a["n_c"],
                             subnet_count=a["subnet_count"])
        assert rc == _lib.B2_EINVAL, kw
        assert all((x == SENTINEL).all() for x in outs), kw
    assert np.array_equal(eng.get_weights(), weights) and eng.get_head(0) == head and eng.tree_size() == len(tree[0])
    fresh = Engine(0)      # no tree
    try:
        rc, outs = _raw_call(fresh, wire, woff, subnets, members, off, EPOCH, cur, cps, spe)
        assert rc == _lib.B2_EINVAL and all((x == SENTINEL).all() for x in outs)
    finally:
        fresh.close()


def test_device_guards(eng):
    spe, cps, size = 8, 4, 5
    tree = OS._tree(spe)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    members, off = OS._committees(spe * cps, size)
    wires, subnets, cur = OS.every_status_case(tree, spe, cps, members, off)
    want = _oracle(wires, subnets, members, off, tree, EPOCH, cur, cps, spe)
    assert eng.guard_flags() == 0
    wire, woff = T._wire(wires)
    w1 = woff.copy()
    w1[1] = w1[2] + 1                                       # row 1 reversed
    got = _single_dev(eng, wires, subnets, members, off, EPOCH, cur, 64, cps, spe, 1, woff=w1)
    assert eng.guard_flags() & 2 and got.status[1] == 1
    w2 = woff.copy()
    w2[-1] = len(wire) + 64                                 # the last row ends past the wire
    got = _single_dev(eng, wires, subnets, members, off, EPOCH, cur, 64, cps, spe, 1, woff=w2)
    assert eng.guard_flags() & 2 and got.status[-1] == 1
    assert np.array_equal(got.status[:-1], want.status[:-1])
    # a malformed committee row: committee 3 * cps + cps - 1 ends past n_sig -> only its placeholder, its members' items status 8
    c = 4 * cps - 1
    bad = off.copy().astype(np.int64)
    bad[c + 1] = bad[-1] + 5
    got = _single_dev(eng, wires, subnets, members, bad.astype(np.uint32), EPOCH, cur, 64, cps, spe, 1)
    assert eng.guard_flags() & 2
    hit = [i for i in range(len(wires)) if want.status[i] in (0, 13) and int.from_bytes(wires[i][0:8], "little") == cps - 1]
    assert hit and all(got.status[i] == 8 for i in hit)
    assert int(got.vote_off[c + 1]) - int(got.vote_off[c]) == 1


# ------------------------------------------------------------------------------------------ full size
def test_full_size_epoch_matches_phase0_intake(eng):
    """2^20 validators (32 slots x 64 committees of 512), two heads per committee, 300 unknown heads, 1 % second items: the two intakes
    on the same votes, and every vote's message against the oracle's signing root"""
    spe, cps, csize, epoch = 32, 64, 512, 5
    n_c = spe * cps
    n = n_c * csize
    rng = np.random.default_rng(2025)
    nb = 64
    parent = np.array([0] + [max(0, b - 1 - int(rng.integers(0, 2))) for b in range(1, nb)], dtype=np.uint32)
    slot = (epoch * spe - 20 + np.arange(nb)).astype(np.uint64)
    roots = np.frombuffer(b"".join(hashlib.sha256(b"single-full%d" % b).digest() for b in range(nb)), np.uint8).reshape(nb, 32).copy()
    eng.tree_load(parent, slot, roots, np.ones(nb, np.uint8))
    start = epoch * spe
    members = rng.permutation(n).astype(np.uint32)
    off = (np.arange(n_c + 1) * csize).astype(np.uint32)
    c = np.repeat(np.arange(n_c), csize)
    p = np.tile(np.arange(csize), n_c)
    s_c = start + np.arange(n_c) // cps
    data = np.zeros((n_c, 2, 128), np.uint8)
    for k in range(n_c):
        ok = np.nonzero(slot <= s_c[k])[0]
        for v in range(2):
            h = int(ok[rng.integers(0, len(ok))])
            t = IO.ancestor(parent, slot, h, start)
            data[k, v] = np.frombuffer(IO.data128(int(s_c[k]), k % cps, bytes(roots[h]), epoch - 1, bytes(roots[0]), epoch, bytes(roots[t])), np.uint8)
    L0 = 228 + csize // 8 + 1
    rec0 = np.zeros((n, L0), np.uint8)
    rec0[:, 0] = 228
    rec0[:, 4:132] = data[c, rng.integers(0, 2, size=n)]
    rec0[:, 132:228] = rng.integers(0, 256, size=(n, 96), dtype=np.uint8)
    rec0[np.arange(n), 228 + p // 8] = (1 << (p % 8)).astype(np.uint8)
    rec0[:, L0 - 1] |= 1
    unknown = rng.choice(n, size=300, replace=False)
    rec0[unknown, 20:52] = rng.integers(0, 256, size=(300, 32), dtype=np.uint8)
    dup = rng.choice(n, size=n // 100, replace=False)
    extra = rec0[dup].copy()
    extra[::2, 4 + 56] ^= 1
    who = np.concatenate([members, members[dup]])
    cc = np.concatenate([c, c[dup]])
    rec0 = np.vstack([rec0, extra])
    order = rng.permutation(rec0.shape[0])
    rec0, who, cc = rec0[order], who[order], cc[order]
    rec1 = np.zeros((rec0.shape[0], 240), np.uint8)
    rec1[:, 0:8] = np.ascontiguousarray(rec0[:, 12:20])
    rec1[:, 8:16] = who.astype("<u8").view(np.uint8).reshape(-1, 8)
    rec1[:, 16:144] = rec0[:, 4:132]
    rec1[:, 24:32] = 0
    rec1[:, 144:240] = rec0[:, 132:228]
    subnets = (cc % 64).astype(np.uint32)       # (cps * (slot % spe) + index) % 64 = c % 64 with c = (slot - start) * cps + index
    cur = (epoch + 1) * spe + 3
    mv = 2 * n_c + 64
    woff0 = (np.arange(rec0.shape[0] + 1, dtype=np.uint64) * L0).astype(np.uint32)
    woff1 = (np.arange(rec1.shape[0] + 1, dtype=np.uint64) * 240).astype(np.uint32)
    p0 = eng.attestation_intake(rec0.tobytes(), woff0, off, epoch, cur, DOMAIN, cps, spe, csize // 8, mv)
    s1 = eng.single_attestation_intake(rec1.tobytes(), woff1, subnets, members, off, epoch, cur, DOMAIN, cps, spe, csize // 8, mv)
    assert {0, 9, 13} <= set(s1.status.tolist())
    assert np.array_equal(p0.status, s1.status)
    for f in ("vote", "vote_off", "sigs", "source_epoch", "target_epoch", "block_idx"):
        assert np.array_equal(getattr(p0, f), getattr(s1, f)), f
    diff = p0.data128 != s1.data128
    assert not diff[:, :8].any() and not diff[:, 16:].any() and not s1.data128[:, 8:16].any()
    k = min(int(s1.vote_off[-1]), mv)
    for v in range(k):
        d = bytes(s1.data128[v])
        want = Spec.compute_signing_root(IO.data_from_bytes(d), DOMAIN) if any(d) else bytes(32)
        assert bytes(s1.msgs[v]) == want, v
    assert eng.guard_flags() == 0


def test_device_form_refusals_change_nothing(eng):
    """the device form refuses what the host form refuses (those it can see) and writes nothing"""
    from pos_evolution_b200 import _lib
    spe, cps, size = 8, 4, 5
    tree = OS._tree(spe)
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    members, off = OS._committees(spe * cps, size)
    wires, subnets, cur = OS.every_status_case(tree, spe, cps, members, off)
    wire, woff = T._wire(wires)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32), device=DEV)      # noqa: E731
    d_wire = torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV)
    d_woff, d_sub, d_mem, d_off = t(woff), t(subnets), t(members), t(off)
    n_att, n_sig, mv = len(wires), int(off[-1]), 16
    outs = [torch.full((n,), SENTINEL, dtype=torch.uint8, device=DEV) for n in (4 * n_att, 4 * n_sig, 4 * len(off), 96 * n_sig, 128 * mv, 32 * mv,
                                                                              8 * mv, 8 * mv, 4 * mv)]
    dom = np.frombuffer(DOMAIN, np.uint8)
    base = dict(sub=d_sub.data_ptr(), count=64, mem=d_mem.data_ptr(), epoch=EPOCH, cur=cur, n_c=spe * cps, stride=1)

    def call(**kw):
        a = dict(base, **kw)
        return eng.lib.b2_single_attestation_intake_dev(eng.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), n_att, a["sub"], a["count"],
                                                        a["mem"], d_off.data_ptr(), a["n_c"], n_sig, cps, spe, a["stride"], a["epoch"], a["cur"],
                                                        _p(dom), mv, *[o.data_ptr() for o in outs], None)
    for kw in (dict(sub=None), dict(mem=None), dict(count=0), dict(epoch=EPOCH + 2), dict(n_c=spe * cps - 1), dict(stride=0), dict(stride=257)):
        assert call(**kw) == _lib.B2_EINVAL, kw
        torch.cuda.synchronize()
        assert all(bool((o == SENTINEL).all()) for o in outs), kw
    assert call() == 0
    torch.cuda.synchronize()
