"""Fork choice (K8 vote scatter, K9 tree phase) at every form b2_get_head / b2_get_weights choose by tree size, on adversarial block
trees, against the numpy oracle (oracle/fast.py: ghost_weights, ghost_viable, ghost_head).  Weights are compared bit for bit as u64,
heads as block indices.  Every get_head also asserts which form ran (form() below mirrors the host code's thresholds), so a moved
threshold fails here instead of leaving a form untested."""
import os

import numpy as np
import pytest

import scenarios
from oracle import fast

gpu = pytest.mark.gpu

# the shared-memory budgets of the host code's tree_form_of: the tree phase (226 KB per block) and the vote bins
TREE_SMEM_BYTES = 226 * 1024
BINS_SMEM_BYTES = 200 * 1024


def form(n):
    """the forms a tree of n blocks runs in:
      smem_tree   tree phase in shared memory (votes/prefix u64[n+1], packed word u32[n], marks u32[n+1], 15 elements per thread at most);
      work_list   ... with the work list u32[n] of the marking phase too;
      maxpt       elements per thread of the shared-memory instantiation (11 up to 11 * 1024 blocks, else 15);
      smem_votes  vote scatter with per-CTA bins in shared memory (k_ghost_votes_smem), else global atomics (k_ghost_votes);
      packed      subtree size and root rank fit the 15-bit fields of the packed word;
      launches    kernels per b2_get_head: 1 (k_get_head_fused) when the tree phase fits shared memory, else 2"""
    smem = 16 * n + 16 <= TREE_SMEM_BYTES and n <= 15 * 1024
    return {"smem_tree": smem, "work_list": smem and 20 * n + 16 <= TREE_SMEM_BYTES, "maxpt": (11 if n <= 11 * 1024 else 15) if smem else None,
            "smem_votes": 8 * n <= BINS_SMEM_BYTES, "packed": n < 32768, "launches": 1 if smem else 2}


def form_row(n):
    """row of the table of forms: 0 fused/MAXPT 11/list, 1 MAXPT 15/list, 2 MAXPT 15/per-parent loop, 3 generic tree + shared-memory bins,
    4 generic tree + global-atomic scatter, 5 the same with subtree sizes beyond the packed 15-bit field"""
    f = form(n)
    if f["smem_tree"]:
        return 0 if f["maxpt"] == 11 else 1 if f["work_list"] else 2
    return 3 if f["smem_votes"] else 4 if f["packed"] else 5


FORM_SIZES = (300, 11400, 14463, 20000, 40000)                  # one tree size per form
RELOAD_SIZES = (300, 11265, 14463, 14464, 25601, 1, 11570)
SWEEP_VARIANTS_BLOCKS = 30000


def test_form_table_edges():
    """the thresholds of form() at the edges of every row, and the sizes of this file reach every row"""
    edges = {1: 0, 11264: 0, 11265: 1, 11570: 1, 11571: 2, 14463: 2, 14464: 3, 25600: 3, 25601: 4, 32767: 4, 32768: 5, 65537: 5}
    assert {n: form_row(n) for n in edges} == edges
    assert 16 * 14463 + 16 == TREE_SMEM_BYTES and 8 * 25600 == BINS_SMEM_BYTES
    assert {form_row(n) for n in FORM_SIZES + RELOAD_SIZES + (SWEEP_VARIANTS_BLOCKS,)} == set(range(6))


# ------------------------------------------------------------------------------------------ fixtures and the checks every case runs
@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng2():
    """a context in the two-launch form of get_head (B2_HEAD_FUSED=0)"""
    from pos_evolution_b200.engine import Engine
    os.environ["B2_HEAD_FUSED"] = "0"
    try:
        e = Engine(0)
    finally:
        del os.environ["B2_HEAD_FUSED"]
    yield e
    e.close()


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Case:
    """one fork-choice world: block tree, registry (effective balance, active / slashed flags) and latest messages, with the
    fork-choice variant (votes older than min_epoch expire; exclude_slashed)"""

    def __init__(self, tree, msg_block, has_msg, equiv, eff, active=None, slashed=None, epoch=None, min_epoch=0, exclude_slashed=False):
        self.parent, self.slot, self.roots, self.leaf_viable = tree
        self.n, self.n_val = len(self.parent), len(eff)
        self.msg_block, self.has_msg, self.equiv = msg_block.astype(np.uint32), has_msg.astype(np.uint8), equiv.astype(np.uint8)
        self.eff = eff.astype(np.uint64)
        self.active = np.ones(self.n_val, dtype=np.uint8) if active is None else active.astype(np.uint8)
        self.slashed = np.zeros(self.n_val, dtype=np.uint8) if slashed is None else slashed.astype(np.uint8)
        self.epoch = np.full(self.n_val, 3, dtype=np.uint64) if epoch is None else epoch.astype(np.uint64)
        self.min_epoch, self.exclude_slashed = min_epoch, exclude_slashed
        self.keep = fast.ghost_viable(self.parent, self.leaf_viable)

    def load(self, e, multi=True):
        from oracle.bls12_381 import G1, g1_compress
        pk = np.tile(np.frombuffer(g1_compress(G1), dtype=np.uint8), (self.n_val, 1))   # fork choice never reads the pubkeys
        e.registry_load(pk, self.eff, (self.active | (self.slashed << 1)).astype(np.uint8))
        e.tree_load(self.parent, self.slot, self.roots, self.leaf_viable)
        e.latest_messages_load(self.epoch, self.msg_block, self.has_msg, self.equiv)
        e.set_fork_choice_params(self.min_epoch, self.exclude_slashed)
        if multi:
            e.fc_exchange_setup(0, 1)

    def counted(self, lo=0, hi=None):
        """the validators of [lo, hi) whose latest message counts"""
        m = (self.has_msg != 0) & (self.epoch >= self.min_epoch)
        m[:lo] = False
        if hi is not None:
            m[hi:] = False
        return m.astype(np.uint8)

    def act(self):
        return self.active & (1 - self.slashed) if self.exclude_slashed else self.active

    def weights(self, boost_idx=-1, boost=0, lo=0, hi=None):
        return fast.ghost_weights(self.parent, self.msg_block, self.counted(lo, hi), self.eff, self.act(), self.equiv, boost_idx, boost)

    def direct(self):
        m = (self.counted() != 0) & (self.act() != 0) & (self.equiv == 0)
        d = np.zeros(self.n, dtype=np.uint64)
        np.add.at(d, self.msg_block[m].astype(np.int64), self.eff[m])
        return d

    def head(self, w, justified=0):
        return fast.ghost_head(self.parent, self.roots, self.keep, w, justified)


def head_witnessed(e, n, justified=0, boost_idx=-1, boost=0, fused=True):
    """get_head, asserting the form that ran: kernel launches (1: k_get_head_fused, 2: scatter + k_ghost_tree) and the phase stamps
    only some forms write -- slot 3 the shared-memory tree phase, slot 8 its work-list marking, slot 16 the one-launch kernel's scatter"""
    f = form(n)
    one = fused and f["smem_tree"]
    e.debug_head_clocks()                                         # reading clears the stamps
    l0 = e.launch_count
    h = e.get_head(justified, boost_idx, boost)
    c = e.debug_head_clocks()
    assert e.launch_count - l0 == (1 if one else 2), (n, fused)
    assert c[15] != 0 and (c[3] != 0) == f["smem_tree"] and (c[8] != 0) == f["work_list"] and (c[16] != 0) == one, (n, fused, c[[3, 8, 15, 16]])
    return h


def split_at(n_val):
    """an odd, so unaligned, validator index inside [0, n_val]"""
    return min(n_val, (n_val // 3) | 1)


def dev_path(e, c, justified, boost_idx, boost, w_want, h_want):
    """b2_vote_weights_range_dev over [0, k) and [k, n_val) into one torch buffer (the direct votes, in pre-order: compared as a
    multiset), then b2_head_from_votes_dev with d_weight; the tree phase leaves the buffer zeroed"""
    import torch
    votes = torch.zeros(c.n, dtype=torch.int64, device="cuda")
    k = split_at(c.n_val)
    e.vote_weights_range_dev(0, k, votes)
    e.vote_weights_range_dev(k, c.n_val, votes)
    torch.cuda.synchronize()
    got = votes.cpu().numpy().view(np.uint64)
    want = c.direct()
    assert np.array_equal(np.sort(got), np.sort(want)) and int(got.sum(dtype=np.uint64)) == int(want.sum(dtype=np.uint64))
    d_head = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    d_weight = torch.zeros(c.n, dtype=torch.int64, device="cuda")
    e.head_from_votes_dev(votes, d_head, justified, boost_idx, boost, d_weight)
    torch.cuda.synchronize()
    assert int(d_head.item()) == h_want
    assert np.array_equal(d_weight.cpu().numpy().view(np.uint64), w_want)
    assert not bool(votes.any().item())


def check(e, c, justified=0, boost_idx=-1, boost=0, e2=None, multi=True, dev=True):
    """every entry path against the oracle: get_weights, get_head (witnessed), get_head on the two-launch context e2, get_head_multi of one
    rank over the whole validator set and over the two halves of an unaligned split (only trees in the shared-memory form: above that it
    must refuse, and the next get_head must still be right), and the _dev path"""
    from pos_evolution_b200._lib import B2Error
    w = c.weights(boost_idx, boost)
    want = c.head(w, justified)
    assert np.array_equal(e.get_weights(boost_idx, boost), w)
    assert head_witnessed(e, c.n, justified, boost_idx, boost) == want
    if e2 is not None:
        assert head_witnessed(e2, c.n, justified, boost_idx, boost, fused=False) == want
    if multi:
        if form(c.n)["smem_tree"]:
            assert e.get_head_multi(0, c.n_val, justified, boost_idx, boost) == want
            k = split_at(c.n_val)
            for lo, hi in ((0, k), (k, c.n_val)):
                assert e.get_head_multi(lo, hi, justified, boost_idx, boost) == c.head(c.weights(boost_idx, boost, lo, hi), justified)
        else:
            with pytest.raises(B2Error):
                e.get_head_multi(0, c.n_val, justified, boost_idx, boost)
            assert head_witnessed(e, c.n, justified, boost_idx, boost) == want
    if dev:
        dev_path(e, c, justified, boost_idx, boost, w, want)
    return want


def fork_case(n_blk, n_val=20000, seed=1, eff=None):
    tree = scenarios.fork_tree(n_blk, seed)
    msg_block, has_msg, equiv, active, eff0 = scenarios.votes(n_val, n_blk, seed)
    return Case(tree, msg_block, has_msg, equiv, eff0 if eff is None else eff, active)


# ------------------------------------------------------------------------------------------ the tests
@gpu
@pytest.mark.parametrize("n_blk", FORM_SIZES)
def test_entry_paths_agree(eng, eng2, n_blk):
    c = fork_case(n_blk, seed=n_blk)
    c.load(eng)
    c.load(eng2, multi=False)
    boost = fast.proposer_boost_score(c.eff, c.active, 32, 40)
    for justified, boost_idx in ((0, -1), (0, n_blk - 1), (n_blk // 3, n_blk // 2)):
        check(eng, c, justified, boost_idx, boost, e2=eng2)


@gpu
@pytest.mark.parametrize("n_blk", FORM_SIZES)
@pytest.mark.parametrize("shape", scenarios.TREE_SHAPES)
def test_tree_shapes(eng, shape, n_blk):
    """chain (at 40 000 blocks subtree sizes beyond 15 bits), star (one parent walking all children), broom, complete binary tree,
    uniform-random parents, comb; every leaf-viability mode; justified block 0 and the deep viable leaf's parent"""
    rng = np.random.default_rng(n_blk + len(shape))
    n_val = 20000
    for seed, viability in enumerate(("random", "none", "deep")):
        tree = scenarios.tree_shape(shape, n_blk, viability, seed)
        msg_block = rng.integers(0, n_blk, size=n_val)
        has_msg = rng.random(n_val) < 0.95
        equiv = rng.random(n_val) < 0.01
        eff = np.where(rng.random(n_val) < 0.9, 32, rng.integers(16, 33, size=n_val)).astype(np.uint64) * np.uint64(10**9)
        c = Case(tree, msg_block, has_msg, equiv, eff, rng.random(n_val) >= 0.01)
        c.load(eng)
        deep = scenarios.deep_side_leaf(c.parent)
        for justified in (0, int(c.parent[deep])):
            check(eng, c, justified, -1, 0, dev=justified == 0)


def _tied_broom(n_blk, roots_kind, winner_viable=True):
    """A broom (chain ending in a fan of leaves) whose fan leaves a < b < c carry the same non-zero weight (equal numbers of validators of
    equal balance).  Roots rank b > a > c, so neither index order nor its reverse picks the winner b; roots_kind: "hash" (unrelated
    roots), "prefix31" (the three share a 31-byte prefix, differ in byte 31), "byte0" (they differ only in byte 0).  With
    winner_viable=False, b is a non-viable leaf and a must win."""
    parent, slot, roots, leaf_viable = scenarios.tree_shape("broom", n_blk, "all", seed=3)
    fan = np.nonzero(parent == parent[-1])[0]
    a, b, c = int(fan[0]), int(fan[len(fan) // 2]), int(fan[-1])
    if roots_kind == "hash":
        hi = sorted(bytes(roots[x]) for x in (a, b, c))
        roots[c], roots[a], roots[b] = (np.frombuffer(r, dtype=np.uint8) for r in hi)
    else:
        base = np.frombuffer(scenarios._h(b"tie" + roots_kind.encode()), dtype=np.uint8)
        at = 31 if roots_kind == "prefix31" else 0
        for x, d in ((c, 0x7f), (a, 0x80), (b, 0x81)):
            roots[x] = base
            roots[x, at] = d
    if not winner_viable:
        leaf_viable[b] = 0
    n_val = 3 * 4000
    msg_block = np.array([a, b, c], dtype=np.uint32)[np.arange(n_val) % 3]
    eff = np.full(n_val, 32 * 10**9, dtype=np.uint64)
    return Case((parent, slot, roots, leaf_viable), msg_block, np.ones(n_val, np.uint8), np.zeros(n_val, np.uint8), eff), a, b, c


@gpu
@pytest.mark.parametrize("n_blk", FORM_SIZES)
def test_ties_and_roots(eng, n_blk):
    for roots_kind in ("hash", "prefix31", "byte0"):
        for winner_viable in (True, False):
            c, a, b, _ = _tied_broom(n_blk, roots_kind, winner_viable)
            assert len({bytes(r) for r in c.roots}) == n_blk
            c.load(eng)
            w = c.weights()
            assert w[a] == w[b] > 0
            assert check(eng, c, dev=False) == (b if winner_viable else a)


def _below(parent, j, b):
    """True iff block b lies in the subtree of block j (topological order: ancestors have smaller indices)"""
    while b > j:
        b = int(parent[b])
    return b == j


@gpu
@pytest.mark.parametrize("n_blk", FORM_SIZES)
def test_weights_boost_and_justified(eng, n_blk):
    """effective balances of 2^32 - 1, 2^32 and 2^32 + 1 Gwei (sums carry across the 32-bit halves); totals above 2^62 (boost
    included, below 2^64); boost_score = 0; the boost on a non-viable block, on the justified block and outside the justified subtree
    (its ancestor block 0, and the deepest block when it lies in another branch); the justified block a leaf, a non-viable block, the
    deepest block and the last block"""
    n_val = 20000
    v = np.arange(n_val, dtype=np.uint64)
    for big, eff, boost in ((False, np.uint64(1 << 32) + v % np.uint64(3) - np.uint64(1), (1 << 32) + 1),
                            (True, np.uint64((1 << 63) // n_val) + v % np.uint64(7), (1 << 62) + 12345)):
        c = fork_case(n_blk, n_val, seed=n_blk + 7, eff=eff)
        c.load(eng)
        total = int(c.direct().astype(object).sum()) + boost
        assert total < (1 << 64) and (total > (1 << 62)) == big
        leaf = np.nonzero(scenarios.leaves(c.parent))[0]
        dead = np.nonzero(~c.keep)[0]
        deepest = int(np.argmax(scenarios.depths(c.parent)))
        check(eng, c, 0, n_blk - 1, 0)                                # boost_score = 0
        check(eng, c, 0, int(dead[0]), boost)                         # boost on a non-viable block
        for jb in (int(leaf[len(leaf) // 2]), int(dead[len(dead) // 2]), deepest, n_blk - 1):
            check(eng, c, jb, jb, boost, dev=jb == deepest)           # boost on the justified block
            for out in {0, deepest} - {jb}:
                if not _below(c.parent, jb, out):
                    check(eng, c, jb, out, boost, multi=False, dev=False)


@gpu
@pytest.mark.parametrize("n_val_kind", ("1", "31", "33", "1025", "sm-1", "sm+1", "4sm+1"))
def test_validator_count_sweep(eng, n_sm, n_val_kind):
    """validator counts around the warp (32), the scatter CTA (1 024) and the persistent grid (n_sm x 1 024) on a shared-memory tree and
    on a tree above 25 600 blocks (global-atomic scatter): all votes on one block (the warp fast path), v mod n_blocks (every lane a
    different block), lane-interleaved filtered validators (inactive, equivocating, expired, slashed), votes on blocks 0 and n-1 only"""
    n_val = {"1": 1, "31": 31, "33": 33, "1025": 1025, "sm-1": n_sm * 1024 - 1, "sm+1": n_sm * 1024 + 1, "4sm+1": 4 * n_sm * 1024 + 1}[n_val_kind]
    v = np.arange(n_val)
    for n_blk in (10000, 30000):
        tree = scenarios.fork_tree(n_blk, 23)
        eff = (np.uint64(32 * 10**9) - (v % 5).astype(np.uint64) * np.uint64(10**9))
        ones, zeros = np.ones(n_val, np.uint8), np.zeros(n_val, np.uint8)
        lane = v % 8
        cases = {"one": Case(tree, np.full(n_val, n_blk // 2), ones, zeros, eff),
                 "mod": Case(tree, v % n_blk, ones, zeros, eff),
                 "filtered": Case(tree, (v * 7919) % n_blk, ones, lane == 3, eff, active=lane != 1, slashed=lane == 7,
                                  epoch=np.where(lane == 5, 1, 3), min_epoch=2, exclude_slashed=True),
                 "ends": Case(tree, np.where(v % 2 == 0, 0, n_blk - 1), ones, zeros, eff)}
        for name, c in cases.items():
            c.load(eng)
            check(eng, c, 0, n_blk - 1, 10**9)
        eng.set_fork_choice_params(0, False)


@gpu
def test_fork_choice_variants_global_scatter(eng):
    """vote expiry, slashed exclusion and on_attester_slashing through k_ghost_votes (a tree above 25 600 blocks)"""
    n_val, n_blk = 6000, SWEEP_VARIANTS_BLOCKS
    assert not form(n_blk)["smem_votes"]
    tree = scenarios.fork_tree(n_blk, 11)
    msg_block, has_msg, equiv, active, eff = scenarios.votes(n_val, n_blk, 11)
    rng = np.random.default_rng(11)
    epochs = rng.integers(1, 9, size=n_val)
    slashed = rng.random(n_val) < 0.05
    for min_epoch, excl in ((0, False), (5, False), (0, True), (7, True)):
        c = Case(tree, msg_block, has_msg, equiv, eff, active, slashed, epochs, min_epoch, excl)
        c.load(eng)
        check(eng, c, 0, n_blk - 1, 10**12)
    c = Case(tree, msg_block, has_msg, equiv, eff, active, slashed, epochs)
    c.load(eng)
    a1 = np.unique(rng.integers(0, n_val, size=500)).astype(np.uint32)
    a2 = np.unique(rng.integers(0, n_val, size=500)).astype(np.uint32)
    eng.on_attester_slashing(a1, a2)
    both = np.intersect1d(a1, a2)
    assert len(both) > 0 and not equiv[both].all()
    c.equiv = equiv.astype(np.uint8).copy()
    c.equiv[both] = 1
    check(eng, c, 0, -1, 0)


@gpu
def test_reloads_on_one_context(eng):
    """tree loads of growing and shrinking size on one context, across every form boundary; every entry path after each load"""
    for i, n_blk in enumerate(RELOAD_SIZES):
        c = fork_case(n_blk, 5000, seed=40 + i)
        c.load(eng)
        check(eng, c, 0, n_blk - 1, 10**11)
