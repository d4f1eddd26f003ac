"""The slasher's ground truth on the CPU (tests/slasher_oracle.py): the brute force and Spec.is_slashable_attestation_data against the
pairs the reference's own predicate calls slashable (tests/golden/literal_slashing.json); "a validator is flagged <=> some ordered
pair of its accepted attestations is slashable"; the acceptance statuses and the moving window; and a sequential model of the device's
span tables (ring of H columns, early-stopping walks) against the brute force, which is what the claim "detection is exact against
everything ever accepted although columns are recycled" rests on before any kernel runs."""
import json
import os
import random

import numpy as np
import pytest

import slasher_oracle as SO

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "literal_slashing.json")) as f:
        return json.load(f)


def test_predicates_match_the_reference_pairs(golden):
    from pos_evolution_b200 import spec as PS
    n_pairs = 0
    for stream in golden["streams"]:
        flat = [a for c in stream["calls"] for a in c["aggregates"]]
        triples = [t[1:] for _, aggs in SO.golden_batches(stream) for t in aggs]
        datas = [PS.AttestationData(a["slot"], a["index"], bytes.fromhex(a["beacon_block_root"]),
                                    PS.Checkpoint(a["source"], bytes.fromhex(a["source_root"])),
                                    PS.Checkpoint(a["target"], bytes.fromhex(a["target_root"]))) for a in flat]
        want = {tuple(p) for p in stream["slashable_pairs"]}
        n_pairs += len(want)
        for i in range(len(flat)):
            assert PS.hash_tree_root_attestation_data(datas[i]) == triples[i][2]
            for j in range(len(flat)):
                assert SO.is_slashable(triples[i], triples[j]) == ((i, j) in want)
                assert bool(PS.Spec.is_slashable_attestation_data(datas[i], datas[j])) == ((i, j) in want)
    assert n_pairs > 500


def test_flagged_iff_some_ordered_pair_is_slashable(golden):
    for stream in golden["streams"]:
        bs = SO.BruteSlasher(golden["n_validators"], golden["history_epochs"], 64, 0)
        flagged, members_of = set(), []
        for cur, aggs in SO.golden_batches(stream):
            bs.advance(cur)
            m, off, bits, src, tgt, roots = SO.batch(aggs)
            status, kind, _, n_flagged = bs.update(m, off, bits, src, tgt, roots)
            assert set(status.tolist()) <= {SO.OK, SO.SOURCE_EXPIRED} and n_flagged == np.count_nonzero(kind)
            flagged |= {int(v) for v in m[kind != 0]}
            members_of += [set(a[0]) if st == SO.OK else set() for a, st in zip(aggs, status)]     # a re-submission can have expired
        by_reference = set()
        for i, j in stream["slashable_pairs"]:
            by_reference |= members_of[i] & members_of[j]
        assert flagged == by_reference == bs.slashable_validators()
    assert by_reference                                        # the last stream does hold offenders


def test_acceptance_statuses_and_window():
    bs = SO.BruteSlasher(4, 8, 2, current_epoch=10)             # window 3 .. 10, two aggregates per target
    r = SO.root_of
    aggs = [([0], 9, 10, r(1)), ([0], 10, 9, r(2)), ([0], 10, 11, r(3)), ([0], 2, 10, r(4)), ([1], 3, 10, r(5)), ([2], 9, 10, r(6)), ([3], 9, 9, r(7))]
    m, off, bits, src, tgt, roots = SO.batch(aggs)
    accept = np.array([1, 1, 1, 1, 1, 1, 0], dtype=np.uint8)
    status, kind, conflict, n_flagged = bs.update(m, off, bits, src, tgt, roots, accept)
    assert status.tolist() == [SO.OK, SO.SOURCE_AFTER_TARGET, SO.TARGET_AHEAD, SO.SOURCE_EXPIRED, SO.OK, SO.COLUMN_FULL, SO.NOT_ACCEPTED]
    assert n_flagged == 0 and not kind.any() and (conflict == SO.NO_TARGET).all()
    assert bs.history[2] == [] and bs.history[3] == []
    # the window moves: source 3 leaves it, epoch 11 becomes a valid target, and the old record still convicts a surround
    bs.advance(11)
    status, kind, conflict, _ = bs.update(*SO.batch([([1], 3, 11, r(8)), ([1], 4, 9, r(9)), ([0], 10, 11, r(3))]))
    assert status.tolist() == [SO.SOURCE_EXPIRED, SO.OK, SO.OK]
    assert kind.tolist() == [0, SO.SURROUNDED, 0] and conflict[1].tolist() == [SO.NO_TARGET, 10]
    with pytest.raises(AssertionError):
        bs.advance(10)


def test_kinds_on_small_cases():
    r = SO.root_of
    bs = SO.BruteSlasher(2, 16, 8, current_epoch=12)
    # same data twice is no double vote; a third root at that target is one, judged against the FIRST attestation
    _, kind, _, _ = bs.update(*SO.batch([([0, 1], 4, 5, r(1)), ([0], 4, 5, r(1)), ([0], 3, 5, r(2)), ([0], 4, 5, r(1))]))
    assert kind.tolist() == [0, 0, 0, SO.DOUBLE, 0]
    # equal sources or equal targets do not surround; inside one call both halves of a surround are flagged, in either position
    _, kind, conflict, _ = bs.update(*SO.batch([([1], 6, 9, r(3)), ([1], 6, 8, r(4)), ([1], 7, 9, r(5))]))
    assert kind.tolist() == [0, 0, SO.DOUBLE]
    _, kind, conflict, _ = bs.update(*SO.batch([([1], 7, 8, r(6)), ([1], 5, 10, r(7))]))
    assert kind.tolist() == [SO.SURROUNDED | SO.DOUBLE, SO.SURROUNDS] and conflict.tolist() == [[SO.NO_TARGET, 10], [8, SO.NO_TARGET]]


class SpanModel:
    """What the kernels of slasher.cuh compute, executed one member at a time: min/max target-span and first-id cells in a ring of H
    columns, walks that stop at the first cell already covered, columns emptied as the window passes them."""

    def __init__(self, n, H, K, cur):
        self.n, self.H, self.K, self.cur = n, H, K, cur
        self.min_span = np.full((n, H), 0xFFFF, dtype=np.int64)
        self.max_span = np.zeros((n, H), dtype=np.int64)
        self.first = np.full((n, H), 0xFFFF, dtype=np.int64)
        self.count = np.zeros(H, dtype=np.int64)
        self.root = {}

    @property
    def low(self):
        return max(0, self.cur - self.H + 1)

    def advance(self, cur):
        for e in range(self.cur + 1, cur + 1) if cur - self.cur < self.H else range(self.H):
            c = e % self.H
            self.min_span[:, c], self.max_span[:, c], self.first[:, c], self.count[c] = 0xFFFF, 0, 0xFFFF, 0
        self.cur = cur

    def update(self, members, off, bits, src, tgt, roots):
        H, n_agg = self.H, len(off) - 1
        status = np.zeros(n_agg, dtype=np.int32)
        ids = [None] * n_agg
        taken = {}
        for a in range(n_agg):
            s, t = int(src[a]), int(tgt[a])
            status[a] = SO.SOURCE_AFTER_TARGET if s > t else SO.TARGET_AHEAD if t > self.cur else SO.SOURCE_EXPIRED if s < self.low else SO.OK
            if status[a] == SO.OK:
                want = int(self.count[t % H]) + taken.get(t, 0)
                taken[t] = taken.get(t, 0) + 1
                if want >= self.K:
                    status[a] = SO.COLUMN_FULL
                else:
                    ids[a] = want
                    self.root[(t % H, want)] = bytes(roots[a])
        slots = lambda a: [(int(off[a]) + j, int(members[off[a] + j])) for j in range(int(off[a + 1] - off[a])) if (bits[a, j >> 3] >> (j & 7)) & 1]  # noqa: E731
        for a in range(n_agg):
            if ids[a] is None:
                continue
            s, t = int(src[a]), int(tgt[a])
            self.count[t % H] = max(self.count[t % H], ids[a] + 1)
            for _, v in slots(a):
                self.first[v, t % H] = min(self.first[v, t % H], ids[a])
                for e in range(s - 1, self.low - 1, -1):
                    if self.min_span[v, e % H] <= t - e:
                        break
                    self.min_span[v, e % H] = t - e
                for e in range(s + 1, t):
                    if self.max_span[v, e % H] >= t - e:
                        break
                    self.max_span[v, e % H] = t - e
        kind = np.zeros(int(off[-1]), dtype=np.uint8)
        conflict = np.full((int(off[-1]), 2), SO.NO_TARGET, dtype=np.uint32)
        for a in range(n_agg):
            if ids[a] is None:
                continue
            s, t = int(src[a]), int(tgt[a])
            for i, v in slots(a):
                if self.root[(t % H, int(self.first[v, t % H]))] != self.root[(t % H, ids[a])]:
                    kind[i] |= SO.DOUBLE
                lo, hi = int(self.min_span[v, s % H]), int(self.max_span[v, s % H])
                if lo != 0xFFFF and s + lo < t:
                    kind[i] |= SO.SURROUNDS
                    conflict[i, 0] = s + lo
                if s + hi > t:
                    kind[i] |= SO.SURROUNDED
                    conflict[i, 1] = s + hi
        return status, kind, conflict, int(np.count_nonzero(kind))


@pytest.mark.parametrize("H,K,seed", [(8, 6, 1), (8, 64, 2), (5, 64, 3), (32, 64, 4), (3, 3, 5)])
def test_span_tables_in_a_ring_equal_the_brute_force(H, K, seed):
    rng = random.Random(seed)
    n, cur = 6, rng.randrange(0, 3)
    bs, model = SO.BruteSlasher(n, H, K, cur), SpanModel(n, H, K, cur)
    flagged = 0
    for _ in range(250):
        cur += rng.choice([0, 0, 1, 1, 2, H - 1, H + 3] if rng.random() < 0.1 else [0, 1])
        bs.advance(cur)
        model.advance(cur)
        aggs = []
        for _ in range(rng.randrange(1, 6)):
            if rng.random() < 0.4:
                s = rng.randrange(max(0, cur - H - 1), cur + 2)
                t = rng.randrange(max(0, s - 1), cur + 2)
            else:
                s, t = max(0, cur - 1), cur
            aggs.append((rng.sample(range(n), rng.randrange(1, 4)), s, t, SO.root_of(rng.randrange(3) if rng.random() < 0.3 else 0)))
        args = SO.batch(aggs)
        want, got = bs.update(*args), model.update(*args)
        for w, g in zip(want, got):
            assert np.array_equal(w, g), (cur, aggs, w, g)
        flagged += want[3]
    assert flagged > 20
