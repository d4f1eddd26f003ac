"""Differential tests: what the reference's own fenced python blocks compute (pos-evolution.md, executed by
tests/golden/gen_golden.py and stored in tests/golden/literal_oracle.json) vs the oracle's restatement vs the numpy
array form.  The inputs are built here, from the same seeds the generator used."""
import copy
import hashlib
import json
import os

import numpy as np
import pytest

import scenarios
from oracle import fast
from oracle import spec as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "literal_oracle.json")
SHUFFLE_CASES = ((1, "a"), (2, "b"), (37, "c"), (256, "d"), (257, "e"), (1000, "f"))
LMD_UPDATES = ((1, 10, [1, 2, 3, 40]), (2, 20, [2, 3, 17, 41, 63]), (1, 30, [2, 50]))      # (target epoch, block, attesting indices)


@pytest.fixture(scope="module")
def env():
    spec, state = scenarios.minimal_state(64, slot=9)
    with open(GOLDEN) as f:
        return spec, state, json.load(f)


def test_shuffle_literal_vs_oracle_vs_numpy(env):
    spec, _, ref = env
    for n, tag in SHUFFLE_CASES:
        seed = hashlib.sha256(tag.encode()).digest()
        lit = ref["shuffle"]["%d/%s" % (n, tag)]
        assert lit == [spec.compute_shuffled_index(i, n, seed) for i in range(n)]
        assert lit == fast.shuffle_permutation(n, seed, spec.p.SHUFFLE_ROUND_COUNT).tolist()
        assert sorted(lit) == list(range(n))


def test_committees_literal_vs_numpy(env):
    spec, state, ref = env
    ref = ref["committees"]
    epoch = 1
    cps = ref["count_per_slot"]
    assert cps == 2 == spec.get_committee_count_per_slot(state, epoch)
    seed = bytes.fromhex(ref["seed"])
    assert seed == spec.get_seed(state, epoch, S.DOMAIN_BEACON_ATTESTER)
    active = np.array(spec.get_active_validator_indices(state, epoch), dtype=np.uint32)
    members, off = fast.committees_for_epoch(active, seed, spec.p.SHUFFLE_ROUND_COUNT, cps, spec.p.SLOTS_PER_EPOCH)
    seen = []
    for s in range(spec.p.SLOTS_PER_EPOCH):
        for c in range(cps):
            lit = ref["committee"]["%d/%d" % (epoch * spec.p.SLOTS_PER_EPOCH + s, c)]
            k = s * cps + c
            assert lit == members[off[k]:off[k + 1]].tolist() == spec.get_beacon_committee(state, 8 + s, c)
            assert len(lit) == 4
            seen += lit
    assert sorted(seen) == list(range(64))          # committees partition the validator set (ref :455)


def _run(fn, state, att):
    st = copy.deepcopy(state)
    try:
        fn(st, att)
        return "ok", st
    except AssertionError:
        return "assert", None


def attestation_cases(spec, state):
    """-> [(attestation, expected outcome)] of test_process_attestation_literal_vs_oracle."""
    cases = [
        scenarios.make_attestation(spec, state, 8, 0),
        scenarios.make_attestation(spec, state, 8, 1, bits=[True, False, True, False]),
        scenarios.make_attestation(spec, state, 5, 1),                                    # previous epoch
        scenarios.make_attestation(spec, state, 8, 0, corrupt="flip_bit"),
        scenarios.make_attestation(spec, state, 8, 0, corrupt="wrong_message"),
        scenarios.make_attestation(spec, state, 8, 1, corrupt="wrong_signer_set"),
        scenarios.make_attestation(spec, state, 8, 0, bits=[False] * 4),                  # empty -> invalid
        scenarios.make_attestation(spec, state, 8, 0, bits=[True] * 3),                   # wrong bit length
    ]
    bad_idx = scenarios.make_attestation(spec, state, 8, 0)
    bad_idx.data = S.AttestationData(8, 2, bad_idx.data.beacon_block_root, bad_idx.data.source, bad_idx.data.target)
    cases.append(bad_idx)                                                                 # index >= committee count
    expect = ["ok", "ok", "ok", "assert", "assert", "assert", "assert", "assert", "assert"]
    return list(zip(cases, expect))


def test_process_attestation_literal_vs_oracle(env):
    spec, state, ref = env
    cases = attestation_cases(spec, state)
    assert len(ref["process_attestation"]) == len(cases)
    for (att, exp), lit in zip(cases, ref["process_attestation"]):
        r_or, st_or = _run(spec.process_attestation, state, att)
        assert lit["result"] == r_or == exp
        if exp == "ok":
            assert lit["current_epoch_participation"] == st_or.current_epoch_participation
            assert lit["previous_epoch_participation"] == st_or.previous_epoch_participation
            assert lit["balances"] == st_or.balances
            assert lit["balances"] != state.balances
    # double inclusion: flags already set -> no second reward
    b1, b2 = ref["double_inclusion_balances"]
    assert b2 == b1
    st = copy.deepcopy(state)
    spec.process_attestation(st, cases[0][0])
    spec.process_attestation(st, cases[0][0])
    assert st.balances == b1


def _small_store(spec, state, n_blocks=200, seed=3):
    parent, slot, roots, leaf_viable = scenarios.fork_tree(n_blocks, seed)
    rb = [bytes(r) for r in roots]
    just = S.Checkpoint(1, rb[0])
    fin = S.Checkpoint(1, rb[0])
    store = S.Store(time=0, genesis_time=0, justified_checkpoint=just, finalized_checkpoint=fin,
                    best_justified_checkpoint=just, proposer_boost_root=rb[n_blocks - 1], equivocating_indices={3, 17})
    has_child = set(int(p) for p in parent[1:])
    for b in range(n_blocks):
        store.blocks[rb[b]] = S.BeaconBlock(int(slot[b]), rb[parent[b]] if b else bytes(32))
        bs = copy.copy(state)
        if b not in has_child and not leaf_viable[b]:
            bs.current_justified_checkpoint = S.Checkpoint(0, b"\x01" * 32)
        else:
            bs.current_justified_checkpoint = just
        bs.finalized_checkpoint = fin
        store.block_states[rb[b]] = bs
    store.checkpoint_states[just] = state
    rng = np.random.default_rng(seed)
    n = len(state.validators)
    for v in range(n):
        if rng.random() < 0.9:
            store.latest_messages[v] = S.LatestMessage(1, rb[int(n_blocks - 1 - min(n_blocks - 1, rng.geometric(0.05)))])
    return store, parent, slot, roots, leaf_viable, rb


def test_get_head_literal_vs_oracle_vs_numpy(env):
    spec, state, ref = env
    state = copy.deepcopy(state)
    state.validators[5].exit_epoch = 0          # inactive validator is not counted
    store, parent, slot, roots, leaf_viable, rb = _small_store(spec, state)
    head_lit = bytes.fromhex(ref["get_head"])
    assert head_lit == spec.get_head(store)
    n = len(state.validators)
    idx_of = {r: i for i, r in enumerate(rb)}
    msg_block = np.zeros(n, dtype=np.uint32)
    has_msg = np.zeros(n, dtype=np.uint8)
    for v, lm in store.latest_messages.items():
        msg_block[v], has_msg[v] = idx_of[lm.root], 1
    eff = np.array([v.effective_balance for v in state.validators], dtype=np.uint64)
    active = np.array([spec.is_active_validator(v, spec.get_current_epoch(state)) for v in state.validators], dtype=np.uint8)
    equiv = np.zeros(n, dtype=np.uint8)
    equiv[list(store.equivocating_indices)] = 1
    boost = fast.proposer_boost_score(eff, active, spec.p.SLOTS_PER_EPOCH, spec.p.PROPOSER_SCORE_BOOST)
    w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, len(rb) - 1, boost)
    for b in range(0, len(rb), 7):
        assert int(w[b]) == spec.get_latest_attesting_balance(store, rb[b])
    keep = fast.ghost_viable(parent, leaf_viable)
    assert set(rb[b] for b in range(len(rb)) if keep[b]) == set(spec.get_filtered_block_tree(store).keys())
    assert rb[fast.ghost_head(parent, roots, keep, w, 0)] == head_lit


def _shape_store(state, parent, slot, roots, leaf_viable, justified, boost_idx, msg_block, has_msg, equiv):
    """A Store holding the block tree of scenarios.tree_shape with store.justified_checkpoint on block `justified`: the leaves that
    leaf_viable marks non-viable carry a different current_justified_checkpoint in their block state (get_filtered_block_tree's test),
    the others the store's.  Latest messages, equivocations and the proposer boost (boost_idx < 0: none) as the array form has them."""
    rb = [bytes(r) for r in roots]
    just = S.Checkpoint(1, rb[justified])
    fin = S.Checkpoint(1, rb[0])
    store = S.Store(time=0, genesis_time=0, justified_checkpoint=just, finalized_checkpoint=fin, best_justified_checkpoint=just,
                    proposer_boost_root=rb[boost_idx] if boost_idx >= 0 else S.ZERO32,
                    equivocating_indices=set(int(v) for v in np.nonzero(equiv)[0]))
    leaf = scenarios.leaves(parent)
    for b in range(len(rb)):
        store.blocks[rb[b]] = S.BeaconBlock(int(slot[b]), rb[parent[b]] if b else bytes(32))
        bs = copy.copy(state)
        bs.current_justified_checkpoint = S.Checkpoint(0, b"\x01" * 32) if leaf[b] and not leaf_viable[b] else just
        bs.finalized_checkpoint = fin
        store.block_states[rb[b]] = bs
    store.checkpoint_states[just] = state
    for v in np.nonzero(has_msg)[0]:
        store.latest_messages[int(v)] = S.LatestMessage(1, rb[msg_block[v]])
    return store


def _shape_cases(shape, n):
    """(viability, justified, boost_idx, votes) combinations of test_fast_vs_spec_on_tree_shapes for one tree shape"""
    parent = scenarios.tree_shape(shape, n)[0]
    leaf = scenarios.leaves(parent)
    inner = [b for b in range(1, n) if not leaf[b]]
    mid = inner[len(inner) // 2] if inner else 0                   # a justified block other than 0 with a subtree below it
    first_leaf = int(np.nonzero(leaf)[0][0])
    return [("random", 0, -1, "random"), ("random", 0, n - 1, "random"), ("random", mid, n - 1, "random"), ("random", mid, mid, "tie"),
            ("all", 0, -1, "tie"), ("all", mid, -1, "tie"), ("all", 0, first_leaf, "tie"), ("none", 0, n - 1, "random"),
            ("none", mid, -1, "tie"), ("deep", 0, -1, "random"), ("deep", 0, -1, "tie"), ("deep", mid, 0, "tie"),
            ("random", first_leaf, -1, "random"), ("deep", n - 1, n - 1, "random")]


def _shape_votes(parent, roots, kind, n_val, justified, rng):
    """random: 90 % of the validators vote for a uniformly drawn block.  tie: the two children of the justified block's first
    multi-child descendant with the highest roots (or of any multi-child block) get the same non-zero weight -- equal numbers of
    validators, all of equal balance (the caller's), voting for blocks inside each child's subtree -- so get_head's root tie-break decides.
    -> (msg_block, has_msg, the tied pair or None)"""
    n = len(parent)
    msg_block = np.zeros(n_val, dtype=np.uint32)
    has_msg = np.zeros(n_val, dtype=np.uint8)
    if kind == "random":
        has_msg[:] = rng.random(n_val) < 0.9
        msg_block[:] = rng.integers(0, n, size=n_val)
        return msg_block, has_msg, None
    children = [[] for _ in range(n)]
    for b in range(1, n):
        children[parent[b]].append(b)
    below = set()
    todo = [justified]
    while todo:
        b = todo.pop()
        below.add(b)
        todo += children[b]
    forks = [b for b in sorted(below) if len(children[b]) >= 2] or [b for b in range(n) if len(children[b]) >= 2]
    if not forks:
        return msg_block, has_msg, None                               # a chain has no siblings: all weights zero
    kids = sorted(children[forks[0]], key=lambda c: bytes(roots[c]))[-2:]
    for side, c in enumerate(kids):
        sub = [c]
        for b in range(c + 1, n):                                    # topological order: a block's subtree lies behind it
            if parent[b] in sub:
                sub.append(b)
        for v in range(side, n_val, 2):
            has_msg[v] = 1
            msg_block[v] = sub[int(rng.integers(0, len(sub)))]
    return msg_block, has_msg, kids


@pytest.mark.parametrize("shape", scenarios.TREE_SHAPES)
def test_fast_vs_spec_on_tree_shapes(env, shape):
    """The numpy array form (fast.ghost_weights / ghost_viable / ghost_head), which the GPU fork-choice tests trust on the adversarial tree
    shapes of scenarios.tree_shape, against the oracle's spec restatement (get_weight / get_filtered_block_tree / get_head) on the same
    trees at 40 blocks: every viability mode, a justified block other than 0 (inner block, leaf, last block), with and without the
    proposer boost (also on the justified block and on a block outside its subtree), and siblings tied at non-zero weight."""
    spec, state0, _ = env
    n, n_val = 40, 64
    rng = np.random.default_rng(len(shape))
    for case, (viability, justified, boost_idx, kind) in enumerate(_shape_cases(shape, n)):
        state = copy.deepcopy(state0)
        parent, slot, roots, leaf_viable = scenarios.tree_shape(shape, n, viability, seed=case)
        if kind == "tie":
            for v in state.validators:
                v.effective_balance = 32 * 10**9
        else:
            state.validators[5].exit_epoch = 0                        # an inactive validator is not counted
        msg_block, has_msg, tied = _shape_votes(parent, roots, kind, n_val, justified, rng)
        equiv = np.zeros(n_val, dtype=np.uint8)
        if kind == "random":
            equiv[[3, 17]] = 1
        eff = np.array([v.effective_balance for v in state.validators], dtype=np.uint64)
        active = np.array([spec.is_active_validator(v, spec.get_current_epoch(state)) for v in state.validators], dtype=np.uint8)
        boost = fast.proposer_boost_score(eff, active, spec.p.SLOTS_PER_EPOCH, spec.p.PROPOSER_SCORE_BOOST) if boost_idx >= 0 else 0
        store = _shape_store(state, parent, slot, roots, leaf_viable, justified, boost_idx, msg_block, has_msg, equiv)
        rb = [bytes(r) for r in roots]
        w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, boost_idx, boost)
        assert [int(x) for x in w] == [spec.get_weight(store, r) for r in rb], (shape, case)
        keep = fast.ghost_viable(parent, leaf_viable)
        filtered = spec.get_filtered_block_tree(store)
        below = {justified}
        for b in range(justified + 1, n):
            if parent[b] in below:
                below.add(b)
        assert set(rb[b] for b in below if keep[b]) == set(filtered.keys()), (shape, case)
        head = fast.ghost_head(parent, roots, keep, w, justified)
        assert rb[head] == spec.get_head(store), (shape, case)
        if tied is not None:                                          # the tie the case was built for is there (before the boost)
            w0 = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, -1, 0)
            assert w0[tied[0]] == w0[tied[1]] > 0, (shape, case)


def test_update_latest_messages_literal_vs_numpy(env):
    spec, state, ref = env
    store, parent, slot, roots, leaf_viable, rb = _small_store(spec, state, n_blocks=50)
    n = len(state.validators)
    idx_of = {r: i for i, r in enumerate(rb)}
    msg_epoch = np.zeros(n, dtype=np.uint64)
    msg_block = np.zeros(n, dtype=np.uint32)
    has_msg = np.zeros(n, dtype=np.uint8)
    for v, lm in store.latest_messages.items():
        msg_epoch[v], msg_block[v], has_msg[v] = lm.epoch, idx_of[lm.root], 1
    equiv = np.zeros(n, dtype=np.uint8)
    equiv[list(store.equivocating_indices)] = 1
    for epoch, blk, idxs in LMD_UPDATES:
        fast.lmd_update(msg_epoch, msg_block, has_msg, equiv, idxs, epoch, blk)
    lit = ref["update_latest_messages"]          # store.latest_messages after the reference applied LMD_UPDATES
    for v in range(n):
        if has_msg[v]:
            assert lit[str(v)] == [int(msg_epoch[v]), rb[msg_block[v]].hex()]
        else:
            assert str(v) not in lit


def test_ffg_literal_vs_oracle(env):
    """process_justification_and_finalization / weigh_justification_and_finalization: the reference's own text (ref :793-852)
    against the oracle's restatement on 80 generated end-of-epoch states; every branch must have fired."""
    spec, state0, ref = env
    seen = set()
    assert len(ref["ffg"]) == 80
    for seed in range(80):
        st_or = scenarios.ffg_case(copy.deepcopy(state0), seed)
        before = (st_or.current_justified_checkpoint, st_or.finalized_checkpoint)
        spec.process_justification_and_finalization(st_or)
        got, want = scenarios.ffg_outcome(st_or), ref["ffg"][seed]
        assert got == want, seed
        justified = S.Checkpoint(want["current_justified"][0], bytes.fromhex(want["current_justified"][1]))
        finalized = S.Checkpoint(want["finalized"][0], bytes.fromhex(want["finalized"][1]))
        seen.add(("justified_changed", justified != before[0]))
        seen.add(("finalized_changed", finalized != before[1]))
        seen.add(("bits", tuple(want["justification_bits"][:2])))
        if finalized != before[1]:
            seen.add(("finalized_distance", spec.get_current_epoch(st_or) - finalized.epoch))
    assert {("justified_changed", True), ("justified_changed", False), ("finalized_changed", True), ("finalized_changed", False)} <= seen
    assert {("bits", (0, 0)), ("bits", (0, 1)), ("bits", (1, 0)), ("bits", (1, 1))} <= seen
    assert {("finalized_distance", 1), ("finalized_distance", 2), ("finalized_distance", 3)} <= seen
