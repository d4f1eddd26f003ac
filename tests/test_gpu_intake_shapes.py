"""The attestation intake (b2_attestation_intake / _dev) and the vote grouping (b2_votes_group_dev, b2_votes_empty_dev) at the shapes
where their one-CTA-per-committee kernels change form: committees of 1 to 2 048 members (MAX_VALIDATORS_PER_COMMITTEE) in ragged
layouts, bit-row strides from 1 to 256, 1 to 2 048 distinct AttestationData or votes per committee (the chunked scans past 256), one
committee per epoch and more than 1 024 of them, and max_votes at, below and above the epoch's vote count.  Every output is compared
with tests/intake_oracle.py or tests/votes_oracle.py, and every output is a view into a larger buffer of sentinel bytes: nothing outside
its declared range may change.  Then an epoch of 2 048-member committees goes from the intake through the vote form of EpochProcessor,
synchronous and pipelined, against the BLS and fork-choice oracle."""
import ctypes
import time

import numpy as np
import pytest
import torch

import intake_oracle as IO
import scenarios
import votes_oracle as VO
from oracle import fast
from oracle.spec import Spec
from oracle.ssz import compute_domain

pytestmark = pytest.mark.gpu

EPOCH = 3
DOMAIN = compute_domain(bytes.fromhex("01000000"), bytes(4), bytes(32))
SENTINEL, PAD = 0xA5, 3
NONE = 0xFFFFFFFF
SIZES = [1, 2, 7, 8, 9, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2047, 2048]
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


class _Padded:
    """n rows of shape `row` and type `dtype` on the device, inside a buffer with PAD more rows of SENTINEL bytes on either side"""

    def __init__(self, n, row=(), dtype=torch.uint8, fill=SENTINEL):
        per = int(np.prod(row)) if row else 1
        self.n, self.isz = n, torch.empty(0, dtype=dtype).element_size()
        self.whole = torch.full(((n + 2 * PAD) * per * self.isz,), SENTINEL, dtype=torch.uint8, device=DEV)
        self.t = self.whole.view(dtype).view(n + 2 * PAD, *row)[PAD:PAD + n]
        if fill != SENTINEL:
            self.t.fill_(fill)

    def unchanged_outside(self, lo, hi):
        """True when no byte outside rows [lo, hi) of the view differs from SENTINEL"""
        b = self.whole.cpu().numpy().reshape(self.n + 2 * PAD, -1)
        return bool((b[:PAD + lo] == SENTINEL).all() and (b[PAD + hi:] == SENTINEL).all())

    def numpy(self):
        return self.t.cpu().numpy()


# ------------------------------------------------------------------------------------------ the intake
def _case(seed, sizes, spe, cps, distinct=2, absent=0.1, dup=0.05, corrupt=0.1, n_blocks=60):
    """(tree, wires, off) of one epoch EPOCH with committees of the given sizes"""
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, n_blocks, max(0, EPOCH * spe - 7))
    wires = IO.ragged_epoch(rng, EPOCH, spe, cps, sizes, tree, distinct=distinct, absent=absent, dup=dup, corrupt=corrupt)
    return tree, wires, IO.ragged_layout(sizes)


def _plain(tree, wires, off, spe, cps, bits_stride, epoch=EPOCH):
    """intake_plain of epoch `epoch` at current slot start_slot(epoch + 1); prints its time (pytest -s)"""
    blocks, ids = IO.block_store(*tree)
    t = time.perf_counter()
    r = IO.intake_plain(wires, off, epoch, (epoch + 1) * spe, DOMAIN, cps, spe, bits_stride, blocks, ids)
    print("intake_plain: %d attestations, committees of up to %d members: %.2f s" % (len(wires), int(np.diff(off).max()), time.perf_counter() - t))
    return r


def _wire(wires):
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    return b"".join(wires), woff


def _check_dev(eng, wires, off, spe, cps, bits_stride, max_votes, want):
    """the device form into sentinel-padded outputs: the oracle's values inside the declared ranges, nothing changed outside them"""
    wire, woff = _wire(wires)
    n_att, n_sig, n_c = len(wires), int(off[-1]), len(off) - 1
    d_wire = torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV)
    d_woff = torch.as_tensor(woff.view(np.int32), device=DEV)
    d_off = torch.as_tensor(np.asarray(off, np.uint32).view(np.int32), device=DEV)
    mv = max_votes
    outs = [_Padded(n_att, dtype=torch.int32), _Padded(n_sig, dtype=torch.int32), _Padded(n_c + 1, dtype=torch.int32), _Padded(n_sig, (96,)),
            _Padded(mv, (128,)), _Padded(mv, (32,)), _Padded(mv, dtype=torch.int64), _Padded(mv, dtype=torch.int64), _Padded(mv, dtype=torch.int32)]
    eng.attestation_intake_dev(d_wire, d_woff, d_off, EPOCH, (EPOCH + 1) * spe, DOMAIN, cps, spe, bits_stride, *[o.t for o in outs])
    torch.cuda.synchronize()
    k = min(int(want.vote_off[-1]), mv)
    for name, o in zip(("status", "vote", "vote_off", "sigs"), outs[:4]):
        assert o.unchanged_outside(0, o.n), name
    for name, o in zip(("data128", "msgs", "source_epoch", "target_epoch", "block_idx"), outs[4:]):
        assert o.unchanged_outside(0, k), name
    a = [o.numpy() for o in outs]
    _assert_equal([a[0], a[1].view(np.uint32), a[2].view(np.uint32), a[3]] + [x[:k] for x in a[4:]], want, k)
    assert eng.guard_flags() == 0


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _check_host(eng, wires, off, spe, cps, bits_stride, max_votes, want):
    """the host form into sentinel-padded host arrays: the oracle's values, zero rows from the epoch's vote count to max_votes, nothing
    changed outside the declared ranges"""
    wire, woff = _wire(wires)
    n_att, n_sig, n_c, mv = len(wires), int(off[-1]), len(off) - 1, max_votes
    spec = [(n_att, 4, np.int32), (n_sig, 4, np.uint32), (n_c + 1, 4, np.uint32), (n_sig, 96, np.uint8), (mv, 128, np.uint8), (mv, 32, np.uint8),
            (mv, 8, np.uint64), (mv, 8, np.uint64), (mv, 4, np.uint32)]
    whole = [np.full((n + 2 * PAD) * b, SENTINEL, np.uint8) for n, b, _ in spec]
    views = [w[PAD * b:(PAD + n) * b] for w, (n, b, _) in zip(whole, spec)]
    w = np.frombuffer(wire, np.uint8)
    rc = eng.lib.b2_attestation_intake(eng.h, _p(w), len(wire), _p(woff), n_att, _p(np.asarray(off, np.uint32)), n_c, cps, spe, bits_stride, EPOCH,
                                       (EPOCH + 1) * spe, _p(np.frombuffer(DOMAIN, np.uint8)), mv, *[_p(v) for v in views])
    assert rc == 0
    for x, (n, b, _) in zip(whole, spec):
        assert (x[:PAD * b] == SENTINEL).all() and (x[(PAD + n) * b:] == SENTINEL).all()
    a = [v.view(dt).reshape(n, -1) if b == 96 or dt == np.uint8 else v.view(dt) for v, (n, b, dt) in zip(views, spec)]
    k = min(int(want.vote_off[-1]), mv)
    for x in a[4:]:
        assert not x[k:].any()
    _assert_equal(a[:4] + [x[:k] for x in a[4:]], want, k)


def _assert_equal(got, want, k):
    status, vote, vote_off, sigs, data, msgs, src, tgt, blk = got
    assert np.array_equal(status, want.status), [(i, int(a), int(b)) for i, (a, b) in enumerate(zip(status, want.status)) if a != b][:10]
    assert np.array_equal(vote_off.astype(np.int64), want.vote_off)
    assert np.array_equal(vote, want.vote)
    assert np.array_equal(sigs, want.sigs)
    for name, g, x in (("data128", data, want.data128), ("msgs", msgs, want.msgs), ("source_epoch", src, want.source_epoch),
                       ("target_epoch", tgt, want.target_epoch), ("block_idx", blk, want.block_idx)):
        assert np.array_equal(g, x[:k]), name


def _both_forms(eng, tree, wires, off, spe, cps, bits_stride, want, max_votes=None):
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    mv = int(want.vote_off[-1]) if max_votes is None else max_votes
    _check_dev(eng, wires, off, spe, cps, bits_stride, mv, want)
    _check_host(eng, wires, off, spe, cps, bits_stride, mv, want)


_CASES = {}


def _ragged(bits_stride):
    """SIZES capped at 8 * bits_stride, one slot per committee; 1-3 distinct data per committee, with absentees, duplicates, failures"""
    if bits_stride not in _CASES:
        sizes = [min(s, 8 * bits_stride) for s in SIZES]
        tree, wires, off = _case(10 + bits_stride, sizes, len(sizes), 1, distinct=[1 + c % 3 for c in range(len(sizes))])
        _CASES[bits_stride] = (tree, wires, off, _plain(tree, wires, off, len(sizes), 1, bits_stride))
    return _CASES[bits_stride]


@pytest.mark.parametrize("bits_stride", [256, 129, 64, 33, 1])
def test_ragged_committees_up_to_2048_members(eng, bits_stride):
    tree, wires, off, want = _ragged(bits_stride)
    assert {0, 13} <= set(want.status.tolist()) and len(set(want.status.tolist())) >= 6
    _both_forms(eng, tree, wires, off, len(SIZES), 1, bits_stride, want)


@pytest.mark.parametrize("below_2048", [True, False])
def test_vote_off_and_every_output_stay_in_bounds(eng, below_2048):
    """An epoch of 32 x 1 committees (n_committees + 1 odd) whose vote_off is a view into a larger buffer: k_intake_scan wrote the
    total one entry past it before the scans took n instead of n + 1 entries.  Up to 2 047 members, or up to 2 048."""
    top = 2047 if below_2048 else 2048
    sizes = [max(1, top >> (c % 12)) for c in range(32)]
    tree, wires, off = _case(5 + top, sizes, 32, 1, distinct=3)
    _both_forms(eng, tree, wires, off, 32, 1, 256, _plain(tree, wires, off, 32, 1, 256))


def _distinct_case():
    """8 committees of 2 048 members (one record length, so intake_numpy applies) with 1, 2, 255, 256, 257, 2 048, 3 and 300 distinct
    data; in the committee of 2 048 every member signs its own data (2 048 groups and votes)"""
    if "distinct" not in _CASES:
        distinct = [1, 2, 255, 256, 257, 2048, 3, 300]
        tree, wires, off = _case(77, [2048] * 8, 4, 2, distinct=distinct, absent=0.0, dup=0.02, corrupt=0.0)
        t = time.perf_counter()
        rec = np.frombuffer(b"".join(wires), np.uint8).reshape(len(wires), -1)
        want = IO.intake_numpy(rec, off.astype(np.int64), EPOCH, (EPOCH + 1) * 4, DOMAIN, 2, 4, 256, *tree)
        print("intake_numpy: %d attestations, committees of 2048 members: %.2f s" % (len(wires), time.perf_counter() - t))
        assert np.diff(want.vote_off).tolist() == distinct
        _CASES["distinct"] = (tree, wires, off, want)
    return _CASES["distinct"]


def test_distinct_data_per_committee_up_to_2048(eng):
    tree, wires, off, want = _distinct_case()
    assert 13 in want.status.tolist()
    _both_forms(eng, tree, wires, off, 4, 2, 256, want)


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_max_votes_around_the_vote_count(eng, delta):
    tree, wires, off, want = _distinct_case()
    _both_forms(eng, tree, wires, off, 4, 2, 256, want, max_votes=int(want.vote_off[-1]) + delta)


def test_single_committee_epoch(eng):
    tree, wires, off = _case(3, [2048], 1, 1, distinct=300, absent=0.2, dup=0.1, corrupt=0.1)
    want = _plain(tree, wires, off, 1, 1, 256)
    assert {0, 13} <= set(want.status.tolist())
    _both_forms(eng, tree, wires, off, 1, 1, 256, want)


def test_more_than_1024_committees(eng):
    """32 slots x 33 committees: k_intake_scan's 1 024 threads take two entries each"""
    rng = np.random.default_rng(4)
    sizes = rng.integers(1, 17, size=32 * 33).tolist()
    tree, wires, off = _case(4, sizes, 32, 33, distinct=2, absent=0.2, dup=0.05, corrupt=0.1)
    want = _plain(tree, wires, off, 32, 33, 2)
    _both_forms(eng, tree, wires, off, 32, 33, 2, want)


# ------------------------------------------------------------------------------------------ the vote grouping
def _votes_epoch(seed, bits_stride):
    """SIZES capped at 8 * bits_stride, vote counts per committee cycling over 1, 255, 256, 257 (a committee of 8 * bits_stride: one
    vote per member, each its own), about 15 % not attesting, committee 3 with nobody attesting; votes nobody attested where a
    committee has more votes than attesters, and its last vote left unattested in every fourth committee"""
    rng = np.random.default_rng(seed)
    cap = 8 * bits_stride
    sizes = [min(s, cap) for s in SIZES]
    nv = [cap if s == cap else (1, 255, 256, 257)[c % 4] for c, s in enumerate(sizes)]
    off = IO.ragged_layout(sizes).astype(np.int64)
    vote_off = np.concatenate([[0], np.cumsum(nv)]).astype(np.int64)
    vote = np.full(int(off[-1]), NONE, dtype=np.int64)
    for c, (s, n) in enumerate(zip(sizes, nv)):
        if c == 3:
            continue
        ids = rng.permutation(s) if n == s == cap else rng.integers(0, max(1, n - (c % 4 == 1)), size=s)
        vote[off[c]:off[c + 1]] = np.where(rng.random(s) < 0.15, NONE, vote_off[c] + ids)
    members = rng.permutation(int(off[-1])).astype(np.uint32)
    sigs = rng.integers(0, 256, size=(int(off[-1]), 96), dtype=np.uint8)
    return off, vote.astype(np.uint32), vote_off, members, sigs


@pytest.mark.parametrize("bits_stride,c_begin,c_end", [(256, 0, 19), (256, 9, 18), (256, 18, 19), (256, 0, 1), (64, 0, 19), (64, 4, 13)])
def test_votes_group_matches_numpy_model(eng, bits_stride, c_begin, c_end):
    off, vote, vote_off, members, sigs = _votes_epoch(20 + bits_stride, bits_stride)
    n_c, n_sig, n_votes = len(off) - 1, int(off[-1]), int(vote_off[-1])
    b0, b1 = int(off[c_begin]), int(off[c_end])
    n_loc = int(vote_off[c_end] - vote_off[c_begin])
    want = VO.group_outputs(members, off, vote, vote_off, sigs[b0:b1], bits_stride, c_begin, c_end)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a).view(np.int32), device=DEV)      # noqa: E731
    o = dict(sigs=_Padded(b1 - b0, (96,)), members=_Padded(n_sig, dtype=torch.int32), pos=_Padded(n_sig, dtype=torch.int32),
             seg=_Padded(n_votes + 1, dtype=torch.int32), bits=_Padded(n_votes, (bits_stride,)), agg=_Padded(n_votes, (bits_stride,)),
             loc=_Padded(n_loc + 1, dtype=torch.int32))
    eng.votes_group_dev(t(vote), t(vote_off.astype(np.uint32)), t(members), t(off.astype(np.uint32)),
                        torch.as_tensor(sigs[b0:b1], device=DEV), c_begin, c_end, o["sigs"].t, o["members"].t, o["pos"].t, o["seg"].t,
                        o["bits"].t, o["agg"].t, o["loc"].t)
    # then b2_votes_empty_dev over aggregates filled with 0x5A: a vote nobody attested gets 96 zero bytes and status 2
    agg_sig, agg_st = _Padded(n_votes, (96,), fill=0x5A), _Padded(n_votes, dtype=torch.int32, fill=7)
    eng.votes_empty_dev(o["bits"].t, agg_sig.t, agg_st.t)
    torch.cuda.synchronize()
    assert eng.guard_flags() == 0
    for k, x in o.items():
        assert x.unchanged_outside(0, x.n), k
    assert agg_sig.unchanged_outside(0, n_votes) and agg_st.unchanged_outside(0, n_votes)
    assert np.array_equal(o["members"].numpy().view(np.uint32), want.members_out)
    assert np.array_equal(o["pos"].numpy(), want.pos_out)
    assert np.array_equal(o["seg"].numpy(), want.seg_off)
    assert np.array_equal(o["loc"].numpy(), want.seg_off_loc)
    assert np.array_equal(o["bits"].numpy(), want.bits)
    assert np.array_equal(o["agg"].numpy(), want.agg_bits)
    assert np.array_equal(o["sigs"].numpy(), want.sigs_out)
    empty = np.bincount(vote[vote != NONE].astype(np.int64), minlength=n_votes) == 0
    assert empty.sum() > n_c and not empty.all()
    assert (agg_sig.numpy()[empty] == 0).all() and (agg_sig.numpy()[~empty] == 0x5A).all()
    assert np.array_equal(agg_st.numpy(), np.where(empty, 2, 7))


# ------------------------------------------------------------------------------------------ end to end at 2 048 members
E2E_SIZES = [2048, 1500, 2048, 700, 1, 257, 2048, 300]
E2E_DISTINCT = [40, 3, 257, 5, 1, 7, 2, 20]
E2E_SPE, E2E_CPS, E2E_STRIDE = 8, 1, 256


def _e2e_world():
    if "e2e" not in _CASES:
        rng = np.random.default_rng(31)
        n_val = sum(E2E_SIZES)
        tree = IO.random_tree(rng, 60, EPOCH * E2E_SPE - 5)
        members = rng.permutation(n_val).astype(np.uint32)
        pks = scenarios.pubkeys(n_val)
        eff = rng.integers(16, 33, size=n_val).astype(np.uint64) * np.uint64(10**9)
        _CASES["e2e"] = (tree, members, IO.ragged_layout(E2E_SIZES), pks, eff)
    return _CASES["e2e"]


def _e2e_epoch(eng, k, tree, members, off):
    """epoch EPOCH + k off the wire, signed by the members' keys (scenarios.secret_key); three kept attestations sign a foreign message
    instead.  Returns (wires, epoch, oracle intake, planted vote ids)."""
    e = EPOCH + k
    rng = np.random.default_rng(40 + k)
    wires = IO.ragged_epoch(rng, e, E2E_SPE, E2E_CPS, E2E_SIZES, tree, distinct=E2E_DISTINCT, absent=0.1, dup=0.02, corrupt=0.02)
    r = _plain(tree, wires, off, E2E_SPE, E2E_CPS, E2E_STRIDE, epoch=e)
    slot_of = []
    for a, w in enumerate(wires):
        c = int.from_bytes(w[4:12], "little") - e * E2E_SPE
        bits = w[228:]
        p = next((8 * i + int(b & -b).bit_length() - 1 for i, b in enumerate(bits) if b), 0)
        slot_of.append(int(off[c]) + p if 0 <= c < len(E2E_SIZES) and p < E2E_SIZES[c] else 0)
    kept = np.nonzero(r.status == 0)[0]
    planted = rng.choice(kept, size=3, replace=False).tolist()
    datas = sorted({bytes(w[4:132]) for w in wires} | {b"foreign"})
    msg = {d: (Spec.compute_signing_root(IO.data_from_bytes(d), DOMAIN) if d != b"foreign" else bytes(32)) for d in datas}
    index = {d: i for i, d in enumerate(datas)}
    msgs = np.frombuffer(b"".join(msg[d] for d in datas), np.uint8).reshape(-1, 32)
    which = [index[b"foreign"] if a in planted else index[bytes(w[4:132])] for a, w in enumerate(wires)]
    sig = eng.sign([scenarios.secret_key(int(members[j])) for j in slot_of], which, msgs)
    wires = [w[:132] + bytes(sig[a]) + w[228:] for a, w in enumerate(wires)]
    for a in kept.tolist():
        r.sigs[slot_of[a]] = sig[a]
    return wires, e, r, sorted({int(r.vote[slot_of[a]]) for a in planted})


@pytest.mark.parametrize("mode", ["sync", "pipelined"])
def test_end_to_end_2048_member_committees(eng, mode):
    from pos_evolution_b200.epoch import EpochProcessor
    tree, members, off, pks, eff = _e2e_world()
    parent, slot, roots = tree
    n_val = len(members)
    if "e2e_epochs" not in _CASES:
        _CASES["e2e_epochs"] = [_e2e_epoch(eng, k, tree, members, off) for k in range(3)]
    epochs = _CASES["e2e_epochs"]
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(*tree, np.ones(len(parent), np.uint8))
    eng.latest_messages_reset()
    mv = sum(E2E_DISTINCT) + len(E2E_SIZES)
    ep = EpochProcessor(eng, len(E2E_SIZES), n_val, E2E_STRIDE, len(parent), device=DEV, depth=3, max_votes=mv)
    ep.set_committees(members, off)
    side = torch.cuda.Stream()
    got, keep = [], []

    def collect(t):
        ok, hd = t.wait()
        got.append((ok.cpu().numpy(), hd, t.aggregate_signatures().cpu().numpy().copy(), t.aggregation_bits().cpu().numpy().copy()))

    for k, (wires, e, r, planted) in enumerate(epochs):
        wire, woff = _wire(wires)
        with torch.cuda.stream(side):
            x = ep.intake_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV),
                              e, (e + 1) * E2E_SPE, DOMAIN, E2E_CPS, E2E_SPE)
        assert np.array_equal(x.status.cpu().numpy(), r.status) and np.array_equal(x.vote_off, r.vote_off)
        keep.append(x)
        if mode == "sync":
            ok, hd = ep.process_epoch_dev(x.sigs, None, x.msgs, x.target_epoch, x.block_idx, votes=(x.vote, x.vote_off))
            torch.cuda.synchronize()
            n = int(x.vote_off[-1])
            s = ep.slots[0]
            got.append((ok.cpu().numpy(), int(hd.item()), s.agg_sig[:n].cpu().numpy().copy(), s.v_aggbits[:n].cpu().numpy().copy()))
        else:
            t = ep.submit_dev(x.sigs, None, x.msgs, x.target_epoch, x.block_idx, last=k == len(epochs) - 1, votes=(x.vote, x.vote_off))
            if t is not None:
                collect(t)
    if mode != "sync":
        for t in ep.drain():
            collect(t)
    assert eng.guard_flags() == 0
    assert len(got) == len(epochs)
    m_epoch, m_block, m_has = np.zeros(n_val, np.uint64), np.zeros(n_val, np.uint32), np.zeros(n_val, np.uint8)
    equiv, active = np.zeros(n_val, np.uint8), np.ones(n_val, np.uint8)
    com = np.repeat(np.arange(len(E2E_SIZES)), E2E_SIZES)
    for k, (wires, e, r, planted) in enumerate(epochs):
        g_ok, g_head, g_agg, g_rows = got[k]
        n = int(r.vote_off[-1])
        attesters = [np.nonzero(r.vote == v)[0] for v in range(n)]
        want_ok = np.array([int(len(a) > 0 and v not in planted) for v, a in enumerate(attesters)], np.uint8)
        assert planted and want_ok[planted].sum() == 0
        assert np.array_equal(g_ok, want_ok), (k, np.nonzero(g_ok != want_ok)[0].tolist())
        for v, a in enumerate(attesters):
            row = np.zeros(8 * E2E_STRIDE, np.uint8)
            row[a - off[com[a]]] = 1
            assert np.array_equal(g_rows[v], np.packbits(row, bitorder="little")), (k, v)
            if want_ok[v]:
                fast.lmd_update(m_epoch, m_block, m_has, equiv, members[a].tolist(), int(r.target_epoch[v]), int(r.block_idx[v]))
        w = fast.ghost_weights(parent, m_block, m_has, eff, active, equiv, -1, 0)
        assert g_head == fast.ghost_head(parent, roots, fast.ghost_viable(parent, np.ones(len(parent), np.uint8)), w, 0), k
        # by linearity, a vote's aggregate is Sign(sum of its attesters' keys, its message): the two largest votes and the smallest
        honest = sorted((v for v in range(n) if v not in planted), key=lambda v: -len(attesters[v]))
        for v in honest[:2] + honest[-1:]:
            a = members[attesters[v]].tolist()
            assert bytes(g_agg[v]) == (scenarios.sign_aggregate(a, bytes(r.msgs[v])) if a else bytes(96)), (k, v)
    e_, b_, h_ = eng.latest_messages_read()
    assert np.array_equal(h_, m_has) and np.array_equal(e_[h_ == 1], m_epoch[h_ == 1]) and np.array_equal(b_[h_ == 1], m_block[h_ == 1])
