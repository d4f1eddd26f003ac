"""The slasher on the GPU (b2_slasher_*: span tables in a ring, kernels of csrc/slasher.cuh) against the brute force of
tests/slasher_oracle.py, byte for byte on status, kind and conflict targets after every call; its device guards and error contract;
and the loop detect -> on_attester_slashing -> get_weight through pos_evolution_b200.spec with real signatures."""
import ctypes
import itertools
import json
import os
import random

import numpy as np
import pytest

import scenarios
import slasher_oracle as SO

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
r = SO.root_of


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


class Twin:
    """one slasher on the device and the brute force beside it; every update is compared"""

    def __init__(self, eng, n, H, K, cur=0):
        eng.slasher_init(n, H, K, cur)
        self.eng, self.bs = eng, SO.BruteSlasher(n, H, K, cur)

    def advance(self, cur):
        self.eng.slasher_advance(cur)
        self.bs.advance(cur)

    def update(self, aggs, accept=None):
        args = SO.batch(aggs)
        got, want = self.eng.slasher_update(*args, accept), self.bs.update(*args, accept)
        for g, w, what in zip(got, want, ("status", "kind", "conflict_target", "n_flagged")):
            assert np.array_equal(g, w), (what, aggs, g, w)
        return got


def test_golden_streams(eng):
    with open(os.path.join(HERE, "golden", "literal_slashing.json")) as f:
        golden = json.load(f)
    for stream in golden["streams"]:
        tw = Twin(eng, golden["n_validators"], golden["history_epochs"], 64)
        flagged, members_of = set(), []
        for cur, aggs in SO.golden_batches(stream):
            tw.advance(cur)
            status, kind, _, _ = tw.update(aggs)
            flagged |= {int(v) for v in SO.batch(aggs)[0][kind != 0]}
            members_of += [set(a[0]) if st == 0 else set() for a, st in zip(aggs, status)]
        by_reference = set()
        for i, j in stream["slashable_pairs"]:
            by_reference |= members_of[i] & members_of[j]
        assert flagged == by_reference


def test_double_votes(eng):
    tw = Twin(eng, 8, 16, 8, cur=6)
    # identical data re-submitted in overlapping aggregates is no double vote
    _, kind, _, n = tw.update([([0, 1, 2], 5, 6, r(1)), ([1, 2, 3], 5, 6, r(1)), ([2], 5, 6, r(1))])
    assert n == 0
    _, kind, _, n = tw.update([([2, 3, 4], 5, 6, r(1))])
    assert n == 0
    # three attestations with one target, the first two sharing a root: only the third is a double vote
    _, kind, _, _ = tw.update([([5], 4, 5, r(7)), ([5], 4, 5, r(7)), ([5, 6], 4, 5, r(8))])
    assert kind.tolist() == [0, 0, SO.DOUBLE, 0]
    _, kind, _, _ = tw.update([([6, 5], 4, 5, r(8)), ([6], 4, 5, r(7))])           # 6 voted r(8) first, 5 voted r(7) first
    assert kind.tolist() == [0, SO.DOUBLE, SO.DOUBLE]


def test_surround_votes(eng):
    tw = Twin(eng, 8, 32, 16, cur=20)
    tw.update([([0], 5, 10, r(1))])
    _, kind, conflict, _ = tw.update([([0], 6, 9, r(2))])                          # surrounded by an earlier call
    assert kind.tolist() == [SO.SURROUNDED] and conflict.tolist() == [[SO.NO_TARGET, 10]]
    _, kind, conflict, _ = tw.update([([0], 4, 11, r(3))])                         # surrounds both
    assert kind.tolist() == [SO.SURROUNDS] and conflict.tolist() == [[9, SO.NO_TARGET]]
    for order in ((0, 1), (1, 0)):                                                 # inside one call, both positions
        pair = [([1 + order[0]], 12, 17, r(4)), ([1 + order[0]], 13, 16, r(5))]
        _, kind, _, _ = tw.update([pair[order[0]], pair[order[1]]])
        assert sorted(kind.tolist()) == [SO.SURROUNDS, SO.SURROUNDED]
    # equal sources or equal targets are no surround; neither is the genesis shape
    _, _, _, n = tw.update([([3], 5, 10, r(1)), ([3], 5, 9, r(2)), ([3], 4, 9, r(2)), ([4], 0, 0, r(6)), ([4], 0, 1, r(6)), ([4], 0, 0, r(6))])
    assert n == 0
    for perm in itertools.permutations([(1, 10), (2, 9), (3, 8)]):                 # nested chain, every order, one call and three calls
        for split in (False, True):
            tw = Twin(eng, 2, 16, 8, cur=12)
            aggs = [([1], s, t, r(t)) for s, t in perm]
            results = [tw.update([a]) for a in aggs] if split else [tw.update(aggs)]
            assert sum(res[3] for res in results) == (2 if split else 3)


@pytest.mark.parametrize("H", [8, 4096])
def test_long_walks_and_the_ring(eng, H):
    cur = 3 * H + 5                                                                # the ring has wrapped
    tw = Twin(eng, 4, H, 64, cur=cur)
    low = cur - H + 1
    tw.update([([0], low, cur, r(1)), ([1], cur, cur, r(1))])                      # the longest max_span walk, and the longest min_span walk
    _, kind, conflict, _ = tw.update([([0], low + 1, cur - 1, r(2)), ([1], low, cur, r(2))])
    assert kind.tolist() == [SO.SURROUNDED, SO.DOUBLE] and conflict[0].tolist() == [SO.NO_TARGET, cur]
    tw.advance(cur + 1)                                                            # by one: `low` is gone
    status, kind, _, _ = tw.update([([2], low, cur + 1, r(3)), ([2], low + 1, cur + 1, r(3)), ([0], low + 2, cur - 2, r(4))])
    assert status.tolist() == [SO.SOURCE_EXPIRED, SO.OK, SO.OK] and kind.tolist() == [0, 0, SO.SURROUNDED]
    # exactness: the older half was recorded more than H/2 epochs before the half that completes the surround
    old = cur + 1
    tw.update([([3], old - 1, old, r(5))])
    c1 = old + H - 3
    tw.advance(c1)
    _, kind, conflict, _ = tw.update([([3], old - 2, c1, r(6))])
    assert kind.tolist() == [SO.SURROUNDS] and conflict[0].tolist() == [old, SO.NO_TARGET]
    c2 = c1 + H - 1
    tw.advance(c2)                                                                 # by H - 1: one column survives
    _, kind, _, _ = tw.update([([3], c1, c2, r(7)), ([3], c1 + 1, c2 - 1, r(8))])
    assert kind.tolist() == [SO.SURROUNDS, SO.SURROUNDED]
    c = c2 + 3 * H
    tw.advance(c)                                                                  # by more than H: every column starts empty
    _, kind, _, n = tw.update([([3], c - 1, c, r(9)), ([0], c - H + 1, c, r(9))])
    assert n == 0
    _, kind, _, _ = tw.update([([0], c - H + 2, c - 1, r(1))])
    assert kind.tolist() == [SO.SURROUNDED]


def test_one_validator_in_64_concurrent_aggregates(eng):
    rng = random.Random(11)
    H, cur = 64, 200
    aggs = []
    for a in range(64):
        s = rng.randrange(cur - H + 1, cur + 1)
        aggs.append(([7] + rng.sample([v for v in range(32) if v != 7], 5), s, rng.randrange(s, cur + 1), r(rng.randrange(4))))
    tw = Twin(eng, 32, H, 128, cur)
    _, kind, conflict, n = tw.update(aggs)
    assert n > 32
    # the surround verdicts of an attestation do not depend on where it stands in the call; "first" (the double vote) may
    perm = list(range(64))
    rng.shuffle(perm)
    tw2 = Twin(eng, 32, H, 128, cur)
    _, kind2, conflict2, _ = tw2.update([aggs[p] for p in perm])
    for new, old in enumerate(perm):
        assert np.array_equal(kind2[6 * new:6 * new + 6] & 6, kind[6 * old:6 * old + 6] & 6)
        assert np.array_equal(conflict2[6 * new:6 * new + 6], conflict[6 * old:6 * old + 6])


def test_random_soak(eng):
    rng = random.Random(5)
    n, H, cur = 64, 16, 3
    tw = Twin(eng, n, H, 64, cur)
    flagged = 0
    for _ in range(200):
        cur += rng.choice([0, 1, 1, 1, 2]) if rng.random() < 0.97 else rng.choice([H - 1, H + 2])
        tw.advance(cur)
        aggs = []
        for _ in range(rng.randrange(1, 9)):
            members = rng.sample(range(n), rng.randrange(1, 17))
            if rng.random() < 0.05:                                                # an offender's span, sometimes outside the window
                s = rng.randrange(max(0, cur - H - 1), cur + 1)
                t = rng.randrange(s, cur + 2)
            else:
                s, t = max(0, cur - 1), cur
            aggs.append((members, s, t, r(cur * 4 + (rng.randrange(1, 4) if rng.random() < 0.05 else 0))))
        accept = np.array([rng.random() < 0.95 for _ in aggs], dtype=np.uint8)
        flagged += tw.update(aggs, accept)[3]
    assert flagged > 50


def test_dev_guards_flag_and_skip(eng):
    import torch
    n, H = 16, 8
    tw = Twin(eng, n, H, 16, cur=10)
    tw.update([([0, 1], 8, 10, r(1))])
    members = np.array([0, 1, 99, 2, 3, 4, 5, 6, 7], dtype=np.uint32)                 # 99: outside the tables
    off = np.array([0, 3, 5, 4, 7, 9], dtype=np.uint32)                             # row 2 runs backwards
    bits = np.full((5, 1), 0xFF, dtype=np.uint8)
    src = np.array([9, 9, 9, 9, 2**32 - 1], dtype=np.uint64)
    tgt = np.array([9, 10, 10, 2**32 - 1, 2**33], dtype=np.uint64)
    roots = np.frombuffer(b"".join(r(k) for k in (2, 3, 4, 5, 6)), dtype=np.uint8).reshape(5, 32)
    want = tw.bs.update(members, off, bits, src, tgt, roots)
    assert want[0].tolist() == [SO.OK, SO.OK, SO.BAD_ROW, SO.TARGET_AHEAD, SO.TARGET_AHEAD] and want[1][:2].tolist() == [SO.SURROUNDED] * 2
    dev = [torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x.view(np.int32) if x.dtype == np.uint32 else x.copy()).cuda()
           for x in (members, off, bits, src, tgt, roots)]
    d_status = torch.full((5,), -1, dtype=torch.int32, device="cuda")
    d_kind = torch.zeros(9, dtype=torch.uint8, device="cuda")
    d_conflict = torch.full((9, 2), -1, dtype=torch.int32, device="cuda")
    d_flagged = torch.zeros(1, dtype=torch.int32, device="cuda")
    eng.guard_flags()
    eng.slasher_update_dev(*dev, None, d_status, d_kind, d_conflict, d_flagged)
    assert eng.guard_flags() == 1 | 2 | 4
    assert np.array_equal(d_status.cpu().numpy(), want[0])
    assert np.array_equal(d_kind.cpu().numpy(), want[1])
    assert np.array_equal(d_conflict.cpu().numpy().view(np.uint32), want[2])
    assert int(d_flagged.item()) == want[3]
    tw.update([([2, 3], 9, 10, r(9)), ([0], 9, 10, r(9))])                          # nothing else was recorded


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def test_failed_host_calls_change_nothing(eng):
    from pos_evolution_b200.engine import Engine
    lib, EINVAL = eng.lib, -1
    fresh = Engine(0)
    m, off, bits, src, tgt, roots = SO.batch([([0, 1], 8, 10, r(1)), ([1, 2], 9, 9, r(2))])
    outs = [np.full(2, 0x5A5A5A5A, dtype=np.int32), np.full(4, 0x5A, dtype=np.uint8), np.full((4, 2), 0x5A5A5A5A, dtype=np.uint32),
            np.full(1, 0x5A5A5A5A, dtype=np.uint32)]
    before = [o.copy() for o in outs]

    def call(h, m=m, off=off, src=src, outs=outs):
        return lib.b2_slasher_update(h, _p(m), _p(off), _p(bits), bits.shape[1], _p(src), _p(tgt), _p(roots), None, 2, *map(_p, outs))

    assert call(fresh.h) == EINVAL and b"b2_slasher_init" in lib.b2_last_error(fresh.h)      # before b2_slasher_init
    assert lib.b2_slasher_advance(fresh.h, 5) == EINVAL
    fresh.close()
    tw = Twin(eng, 4, 8, 8, cur=10)
    tw.update([([0], 9, 10, r(3))])
    assert call(eng.h, off=np.array([0, 3, 2], dtype=np.uint32)) == EINVAL                   # decreasing offsets
    assert call(eng.h, m=np.array([0, 1, 1, 4], dtype=np.uint32)) == EINVAL                  # member outside the tables
    assert call(eng.h, src=np.array([8, 2**32 - 1], dtype=np.uint64)) == EINVAL              # epoch that does not fit 32 bits
    for k in (0, 1, 3):                                                                      # NULL outputs (conflict targets may be NULL)
        assert call(eng.h, outs=[None if i == k else o for i, o in enumerate(outs)]) == EINVAL
    assert lib.b2_slasher_advance(eng.h, 9) == EINVAL                                        # backwards
    assert lib.b2_slasher_init(eng.h, 4, 0, 8, 0) == EINVAL and lib.b2_slasher_init(eng.h, 4, 8, 65536, 0) == EINVAL
    assert all(np.array_equal(o, b) for o, b in zip(outs, before))
    _, kind, _, _ = tw.update([([0, 1], 8, 10, r(1)), ([1, 2], 9, 9, r(2)), ([0], 10, 10, r(4))])   # equals the untouched brute force
    assert kind.tolist() == [SO.DOUBLE, SO.SURROUNDS, SO.SURROUNDED, 0, SO.DOUBLE]


def test_column_full_and_refused_allocation(eng):
    from pos_evolution_b200._lib import B2_ENOMEM, B2Error
    tw = Twin(eng, 4, 8, 2, cur=5)
    status, _, _, _ = tw.update([([0], 4, 5, r(1)), ([1], 4, 5, r(1)), ([2], 4, 5, r(2)), ([0], 3, 4, r(1))])
    assert status.tolist() == [0, 0, SO.COLUMN_FULL, 0]
    status, _, _, _ = tw.update([([0], 4, 5, r(9))])
    assert status.tolist() == [SO.COLUMN_FULL]
    with pytest.raises(B2Error) as e:                        # 6 * 2^24 * 65 535 bytes = 6.6 TB: refused by arithmetic, nothing is allocated
        eng.slasher_init(1 << 24, 65535, 16, 0)
    assert e.value.code == B2_ENOMEM
    status, kind, _, _ = tw.update([([0], 2, 5, r(9)), ([2], 4, 4, r(3))])     # the previous slasher still answers
    assert status.tolist() == [SO.COLUMN_FULL, 0]
    tw.advance(6)
    _, kind, _, _ = tw.update([([0], 2, 6, r(9))])
    assert kind.tolist() == [SO.SURROUNDS]
    eng.slasher_free()
    with pytest.raises(B2Error):
        eng.slasher_update(*SO.batch([([0], 2, 6, r(9))]))


def test_a_context_without_a_slasher_launches_what_it_did(eng):
    from pos_evolution_b200.engine import Engine
    other = Engine(0)
    pk = other.sk_to_pk([1, 2, 3, 4])
    deltas = []
    for e, with_slasher in ((other, False), (eng, True)):
        e.registry_load(pk, np.full(4, 32 * 10**9, dtype=np.uint64))
        if with_slasher:
            e.slasher_init(4, 8, 8, 3)
        c0 = e.launch_count
        e.latest_messages_update([0, 1, 2, 3], [0, 4], np.array([[0x0F]], dtype=np.uint8), [1], [0])
        deltas.append(e.launch_count - c0)
    assert deltas[0] == deltas[1] == 2
    c0 = eng.launch_count
    eng.slasher_update(*SO.batch([([0, 1], 2, 3, r(1))]))
    assert eng.launch_count - c0 == 3                        # k_slasher_rows, k_slasher_record, k_slasher_check
    other.close()


def test_detect_slash_and_discount_end_to_end():
    """two conflicting aggregates with real signatures -> find_attester_slashings -> on_attester_slashing -> get_weight drops"""
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from test_gpu_spec import _state_to_product
    ospec, ostate = scenarios.minimal_state(64, slot=9)
    pspec = PS.Spec(PS.MINIMAL, engine=Engine(0))
    eng = pspec.engine
    state = _state_to_product(PS, ostate)
    committee = [int(v) for v in pspec.get_beacon_committee(state, 8, 0)]
    blocks = {b"\x01" * 32: PS.BeaconBlock(1, state.current_justified_checkpoint.root), b"\x02" * 32: PS.BeaconBlock(1, state.current_justified_checkpoint.root)}

    def signed(data, signers):
        msg = np.frombuffer(pspec.compute_signing_root(data, pspec.get_domain(state, PS.DOMAIN_BEACON_ATTESTER, data.target.epoch)), dtype=np.uint8)
        sigs = eng.sign([scenarios.secret_key(v) for v in signers], [0] * len(signers), msg.reshape(1, 32))
        agg, st = eng.aggregate(sigs, [0, len(signers)])
        assert st[0] == 0
        return PS.IndexedAttestation(sorted(signers), data, agg[0].tobytes())

    just = state.current_justified_checkpoint
    data = [PS.AttestationData(8, 0, head, just, PS.Checkpoint(1, b"\x0a" * 32)) for head in blocks]
    first, second = signed(data[0], committee), signed(data[1], committee[:2])
    forged = PS.IndexedAttestation(sorted(committee), data[1], first.signature)
    pspec.slasher_start(state, history_epochs=8)
    assert pspec.find_attester_slashings(state, [first]) == []
    assert pspec.find_attester_slashings(state, [forged, first]) == []              # a bad signature records nothing; a repeat is no conflict
    found = pspec.find_attester_slashings(state, [second])
    assert len(found) == 1 and found[0].attestation_1 is first and found[0].attestation_2 is second
    store = PS.Store(0, 0, just, just, just, PS.ZERO32, set())
    store.blocks[just.root] = PS.BeaconBlock(0, bytes(32))
    store.blocks.update(blocks)
    for root in store.blocks:
        store.block_states[root] = state
    store.checkpoint_states[just] = state
    for v in committee:
        store.latest_messages[v] = PS.LatestMessage(1, b"\x01" * 32)
    before = pspec.get_weight(store, b"\x01" * 32)
    assert before == sum(state.validators[v].effective_balance for v in committee)
    pspec.on_attester_slashing(store, found[0])
    assert store.equivocating_indices == set(committee[:2])
    assert pspec.get_weight(store, b"\x01" * 32) == before - sum(state.validators[v].effective_balance for v in committee[:2])
    eng.close()
