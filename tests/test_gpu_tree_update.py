"""The block tree changed on the device (b2_tree_add / b2_tree_prune / b2_tree_set_viable): after every change the context must behave
exactly like a fresh b2_tree_load of the resulting arrays -- weights, heads at several justified blocks, tie-breaks, kernel form -- and
the latest messages must be re-mapped through the prune map.  Checked against a second Engine loaded from a host model and against
oracle.fast."""
import numpy as np
import pytest

import scenarios
from oracle import fast

gpu = pytest.mark.gpu
DROP = 0xFFFFFFFF
INF_PK = bytes([0xC0]) + bytes(47)          # the compressed point at infinity: decodable, fails KeyValidate; fork choice never reads it


class Model:
    """The host form of the tree and the latest-message table, changed by the same operations as the device."""

    def __init__(self, parent, roots, viable, n_val, seed=0):
        self.parent = np.asarray(parent, dtype=np.uint32).copy()
        self.roots = np.asarray(roots, dtype=np.uint8).reshape(-1, 32).copy()
        self.viable = np.asarray(viable, dtype=np.uint8).copy()
        rng = np.random.default_rng(seed)
        self.eff = (rng.integers(1, 33, n_val) * 10**9).astype(np.uint64)
        self.epoch = np.zeros(n_val, dtype=np.uint64)
        self.block = np.zeros(n_val, dtype=np.uint32)
        self.has = np.zeros(n_val, dtype=np.uint8)
        self.equiv = np.zeros(n_val, dtype=np.uint8)

    @property
    def n(self):
        return len(self.parent)

    def add(self, parent, roots, viable):
        self.parent = np.concatenate([self.parent, np.asarray(parent, dtype=np.uint32)])
        self.roots = np.vstack([self.roots, np.asarray(roots, dtype=np.uint8).reshape(-1, 32)])
        self.viable = np.concatenate([self.viable, np.asarray(viable, dtype=np.uint8)])

    def prune(self, r):
        kept = np.zeros(self.n, dtype=bool)
        kept[r] = True
        for b in range(r + 1, self.n):
            kept[b] = kept[self.parent[b]]
        mp = np.full(self.n, DROP, dtype=np.uint32)
        mp[kept] = np.arange(int(kept.sum()), dtype=np.uint32)
        parent = mp[self.parent[kept]]
        parent[0] = 0
        self.parent, self.roots, self.viable = parent, self.roots[kept], self.viable[kept]
        old = self.block < len(mp)
        self.block[old] = mp[self.block[old]]
        return mp

    def vote(self, members, target_epoch, block):
        fast.lmd_update(self.epoch, self.block, self.has, self.equiv, members, target_epoch, block)

    def weights(self, boost_idx=-1, boost=0):
        has = self.has * (self.block < self.n)
        return fast.ghost_weights(self.parent, np.where(has != 0, self.block, 0), has, self.eff, np.ones(len(has), np.uint8), self.equiv,
                                  boost_idx, boost)

    def head(self, justified, boost_idx=-1, boost=0):
        return fast.ghost_head(self.parent, self.roots, fast.ghost_viable(self.parent, self.viable), self.weights(boost_idx, boost), justified)


def engine(model):
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    n_val = len(model.eff)
    e.registry_load(np.frombuffer(INF_PK * n_val, dtype=np.uint8).reshape(n_val, 48), model.eff)
    return e


def load(e, model):
    e.tree_load(model.parent, np.zeros(model.n, dtype=np.uint64), model.roots, model.viable)
    e.latest_messages_load(model.epoch, model.block, model.has, model.equiv)


def vote(e, model, members, target_epoch, block):
    members = np.asarray(members, dtype=np.uint32)
    bits = np.packbits(np.ones(len(members), dtype=np.uint8), bitorder="little").reshape(1, -1)
    e.latest_messages_update(members, [0, len(members)], bits, [target_epoch], [block])
    model.vote(members, target_epoch, block)


def justified_ids(model, rng):
    return sorted({0, model.n - 1, int(model.parent[-1]), int(rng.integers(model.n))})


def check(e, ref, model, rng, oracle=True):
    """e (changed in place) against ref (a fresh load of the model) and, when oracle is set, against oracle.fast"""
    load(ref, model)
    assert e.tree_size() == ref.tree_size() == model.n
    boost_idx = int(rng.integers(model.n))
    for bi, bs in ((-1, 0), (boost_idx, 7 * 10**9)):
        w = e.get_weights(bi, bs)
        assert np.array_equal(w, ref.get_weights(bi, bs))
        if oracle:
            assert np.array_equal(w, model.weights(bi, bs))
        for j in justified_ids(model, rng):
            h = e.get_head(j, bi, bs)
            assert h == ref.get_head(j, bi, bs), (j, bi)
            if oracle:
                assert h == model.head(j, bi, bs), (j, bi)
    got, want = e.latest_messages_read(), ref.latest_messages_read()
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def new_blocks(model, rng, k, within=False, tag=0):
    """k blocks with parents biased to recent blocks; within: some parent earlier blocks of the same batch"""
    n = model.n
    parent = np.empty(k, dtype=np.uint32)
    for j in range(k):
        hi = n + j if within else n
        back = int(rng.geometric(0.3)) - 1
        parent[j] = max(0, hi - 1 - back) if rng.random() < 0.8 else int(rng.integers(hi))
    roots = rng.integers(0, 256, (k, 32), dtype=np.uint8)
    roots[:, 0] = tag
    viable = (rng.random(k) >= 0.1).astype(np.uint8)
    return parent, roots, viable


def subtree_sizes(model):
    size = np.ones(model.n, dtype=np.int64)
    for b in range(model.n - 1, 0, -1):
        size[model.parent[b]] += size[b]
    return size


def deep_block(model):
    depth = np.zeros(model.n, dtype=np.int64)
    for b in range(1, model.n):
        depth[b] = depth[model.parent[b]] + 1
    return int(np.argmax(depth))


@gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_random_sequences_match_a_fresh_load(seed):
    run_sequence(seed, 200)


@gpu
def test_random_sequence_generic_form():
    """the multi-CTA insert on a random fork tree above 14 463 blocks: mixed batches whose ancestors and shifted blocks interleave"""
    run_sequence(3, 15_000)


def run_sequence(seed, n_blocks):
    rng = np.random.default_rng(seed)
    n_val = 4096
    p, s, r, v = scenarios.fork_tree(n_blocks, seed)
    model = Model(p, r, v, n_val, seed)
    e, ref = engine(model), engine(model)
    load(e, model)
    vote(e, model, rng.choice(n_val, 1500, replace=False), 1, int(rng.integers(model.n)))
    check(e, ref, model, rng)
    ops = ["add1", "add3", "add32", "vote", "viable", "add500", "vote", "prune_deep", "add32w", "vote", "prune_root", "add3", "viable",
           "prune_leaf", "add32w", "vote", "add1"]
    epoch = 2
    for op in ops:
        if op.startswith("add"):
            k = int(op[3:].rstrip("w"))
            par, roots, via = new_blocks(model, rng, k, within=op.endswith("w"), tag=epoch)
            e.tree_add(par, np.zeros(k, dtype=np.uint64), roots, via)
            model.add(par, roots, via)
        elif op == "vote":
            for _ in range(3):
                vote(e, model, rng.choice(n_val, 700, replace=False), epoch, int(rng.integers(model.n - min(model.n, 40), model.n)))
                epoch += 1
        elif op == "viable":
            idx = rng.choice(model.n, min(model.n, 25), replace=False).astype(np.uint32)
            val = (rng.random(len(idx)) < 0.5).astype(np.uint8)
            e.tree_set_viable(idx, val)
            model.viable[idx] = val
        else:
            root = {"prune_deep": lambda: int(model.parent[deep_block(model)]), "prune_root": lambda: 0, "prune_leaf": lambda: model.n - 1}[op]()
            assert np.array_equal(e.tree_prune(root), model.prune(root))
        check(e, ref, model, rng)


@gpu
@pytest.mark.parametrize("shape", ["chain", "star", "deep"])
def test_form_switches(shape):
    """across the shared-memory tree phase (14 463 blocks) and the shared-memory bins (25 600), up and back down"""
    rng = np.random.default_rng(7)
    n_val = 2048
    p, s, r, v = scenarios.tree_shape("comb" if shape == "deep" else shape, 14_000, viability="deep" if shape == "deep" else "random")
    model = Model(p, r, v, n_val)
    e, ref = engine(model), engine(model)
    load(e, model)
    vote(e, model, np.arange(n_val // 2), 1, model.n - 1)
    for k in (400, 100, 11_200):                        # 14 400 (shared memory), 14 500 (generic tree, smem bins), 25 700 (generic bins)
        if shape == "star":
            par = np.zeros(k, dtype=np.uint32)
        else:
            par = np.arange(model.n - 1, model.n - 1 + k, dtype=np.uint32)
        roots = rng.integers(0, 256, (k, 32), dtype=np.uint8)
        e.tree_add(par, np.zeros(k, dtype=np.uint64), roots, np.ones(k, dtype=np.uint8))
        model.add(par, roots, np.ones(k, dtype=np.uint8))
        vote(e, model, np.arange(n_val // 2, n_val // 2 + 100 + k // 100), 2 + k, model.n - 1)
        check(e, ref, model, rng, oracle=model.n < 20_000)
    size = subtree_sizes(model)
    root = int(np.argmax(np.where(size <= 14_000, size, 0)))      # the largest subtree below both thresholds (a leaf of the star)
    assert np.array_equal(e.tree_prune(root), model.prune(root))
    check(e, ref, model, rng)


@gpu
def test_root_ties():
    """equal roots: the tie-break is the (root, id) order of b2_tree_load; new roots before, between, after and equal to existing ones"""
    rng = np.random.default_rng(3)
    n_val = 512
    roots = np.zeros((5, 32), dtype=np.uint8)
    roots[:, 0] = [0x40, 0x40, 0x80, 0x80, 0x80]
    model = Model([0, 0, 0, 0, 0], roots, np.ones(5), n_val)
    e, ref = engine(model), engine(model)
    load(e, model)
    check(e, ref, model, rng, oracle=False)
    for first in (0x00, 0x40, 0x60, 0x80, 0xFF, 0x40):
        nr = np.zeros((2, 32), dtype=np.uint8)
        nr[:, 0] = first
        e.tree_add([0, 0], np.zeros(2, dtype=np.uint64), nr, [1, 1])
        model.add([0, 0], nr, [1, 1])
        check(e, ref, model, rng, oracle=False)
    assert np.array_equal(e.tree_prune(0), model.prune(0))
    check(e, ref, model, rng, oracle=False)


@gpu
def test_full_size_remap():
    """2^20 validators on a 10 000-block fork tree; a prune that drops about a third of the votes re-maps the table exactly"""
    rng = np.random.default_rng(11)
    n_val = 1 << 20
    p, s, r, v = scenarios.fork_tree(10_000)
    model = Model(p, r, v, n_val)
    e, ref = engine(model), engine(model)
    model.epoch[:] = rng.integers(1, 100, n_val)
    model.block[:] = rng.integers(0, model.n, n_val)
    model.has[:] = rng.random(n_val) < 0.9
    load(e, model)
    size = subtree_sizes(model)
    root = int(np.argmin(np.abs(size - 2 * model.n // 3)))
    mp = e.tree_prune(root)
    assert np.array_equal(mp, model.prune(root))
    dropped = np.count_nonzero((model.has != 0) & (model.block == DROP)) / np.count_nonzero(model.has)
    assert 0.2 < dropped < 0.45
    got = e.latest_messages_read()
    assert np.array_equal(got[0], np.where(model.has != 0, model.epoch, 0))
    assert np.array_equal(got[1], np.where(model.has != 0, model.block, 0))
    assert np.array_equal(got[2], model.has)
    check(e, ref, model, rng)


@gpu
def test_rejected_calls_change_nothing():
    from pos_evolution_b200._lib import B2Error
    rng = np.random.default_rng(5)
    p, s, r, v = scenarios.fork_tree(300)
    model = Model(p, r, v, 1024)
    e, ref = engine(model), engine(model)
    with pytest.raises(B2Error):                          # no tree loaded
        e.tree_add([0], [0], np.zeros((1, 32), np.uint8), [1])
    with pytest.raises(B2Error):
        e.tree_set_viable([0], [1])
    with pytest.raises(B2Error):
        e.tree_prune(0)
    load(e, model)
    vote(e, model, np.arange(600), 1, 250)
    before = (e.get_weights(), e.get_head(0), e.latest_messages_read(), e.tree_size())
    bad = [lambda: e.tree_add([], [], np.zeros((0, 32), np.uint8), []),                                    # k = 0
           lambda: e.tree_add([0, 301], [0, 0], np.zeros((2, 32), np.uint8), [1, 1]),                     # parent == own id
           lambda: e.tree_add([5, 400], [0, 0], np.zeros((2, 32), np.uint8), [1, 1]),                     # parent > own id
           lambda: e.tree_prune(300),
           lambda: e.tree_set_viable([], []),
           lambda: e.tree_set_viable([3, 300], [0, 0])]
    for call in bad:
        n_blocks = e.n_blocks
        with pytest.raises(B2Error):
            call()
        e.n_blocks = n_blocks
        after = (e.get_weights(), e.get_head(0), e.latest_messages_read(), e.tree_size())
        assert np.array_equal(after[0], before[0]) and after[1] == before[1] and after[3] == before[3]
        for a, b in zip(after[2], before[2]):
            assert np.array_equal(a, b)
    check(e, ref, model, rng)


@gpu
def test_nvlink_head_refuses_after_a_size_change():
    from pos_evolution_b200._lib import B2Error
    rng = np.random.default_rng(6)
    p, s, r, v = scenarios.fork_tree(500)
    model = Model(p, r, v, 2048)
    e = engine(model)
    load(e, model)
    vote(e, model, np.arange(1000), 1, 480)
    e.fc_exchange_setup(0, 1)
    assert e.get_head_multi(0, 2048, 0) == e.get_head(0)
    par, roots, via = new_blocks(model, rng, 3)
    e.tree_add(par, np.zeros(3, dtype=np.uint64), roots, via)
    model.add(par, roots, via)
    with pytest.raises(B2Error):
        e.get_head_multi(0, 2048, 0)
    e.fc_exchange_setup(0, 1)
    assert e.get_head_multi(0, 2048, 0) == e.get_head(0) == model.head(0)
    e.tree_prune(int(model.parent[deep_block(model)]))
    with pytest.raises(B2Error):
        e.get_head_multi(0, 2048, 0)


@gpu
def test_epoch_processor_tree_changes():
    import torch
    from pos_evolution_b200.epoch import EpochProcessor
    rng = np.random.default_rng(8)
    p, s, r, v = scenarios.fork_tree(400)
    model = Model(p, r, v, 4096)
    e = engine(model)
    load(e, model)
    ep = EpochProcessor(e, 4, 16, 1, model.n, depth=2)
    vote(e, model, np.arange(2000), 1, 390)
    assert ep.get_head() == e.get_head(0) == model.head(0)
    par, roots, via = new_blocks(model, rng, 40, within=True)
    ep.add_blocks(par, np.zeros(40, dtype=np.uint64), roots, via)
    model.add(par, roots, via)
    assert ep.d_votes.numel() == model.n
    vote(e, model, np.arange(1000, 3000), 2, model.n - 1)
    assert ep.get_head() == model.head(0)
    root = int(model.parent[deep_block(model)])
    assert np.array_equal(ep.prune_tree(root), model.prune(root))
    assert ep.d_votes.numel() == model.n
    ep.set_viable([model.n - 1], [0])
    model.viable[model.n - 1] = 0
    assert ep.get_head() == model.head(0)
    fresh = engine(model)
    load(fresh, model)
    ep2 = EpochProcessor(fresh, 4, 16, 1, model.n, depth=2)
    assert ep.get_head() == ep2.get_head()
    torch.cuda.synchronize()
    p2, s2, r2, v2 = scenarios.fork_tree(model.n + 10)               # a larger tree loaded behind the processor's back
    e.tree_load(p2, s2, r2, v2)
    with pytest.raises(ValueError):
        ep.get_head()
