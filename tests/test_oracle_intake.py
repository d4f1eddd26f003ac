"""CPU checks of the attestation intake's oracle (tests/intake_oracle.py): its tree statuses 9-12 against Spec.validate_on_attestation,
its grouping against a hand-built vote form, and the numpy form against the plain one."""
import numpy as np
import pytest

import intake_oracle as IO
from pos_evolution_b200 import spec as PS

SPE, CPS, CSIZE = 8, 2, 7
DOMAIN = bytes(range(32))


def _layout(csize=CSIZE):
    return np.arange(SPE * CPS + 1, dtype=np.int64) * csize


def _epoch(seed, epoch=3, n_blocks=30, n_extra=20, corrupt=0.4):
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, n_blocks, epoch * SPE - 9)
    wires = IO.random_epoch(rng, epoch, SPE, CPS, CSIZE, tree, n_extra=n_extra, corrupt=corrupt)
    return tree, wires


def test_tree_statuses_agree_with_validate_on_attestation():
    seen = set()
    for seed in range(6):
        seen |= _check_against_spec(seed)
    assert {0, 9, 10, 11, 12, 13} <= seen


def _check_against_spec(seed):
    epoch = 3
    tree, wires = _epoch(seed, epoch)
    blocks, ids = IO.block_store(*tree)
    current_slot = (epoch + 1) * SPE + 2
    r = IO.intake_plain(wires, _layout(), epoch, current_slot, DOMAIN, CPS, SPE, 1, blocks, ids)
    sp = PS.Spec(PS.MINIMAL, engine=object())
    assert sp.p.SLOTS_PER_EPOCH == SPE
    cp = PS.Checkpoint()
    store = PS.Store(time=current_slot * getattr(sp.p, "SECONDS_PER_SLOT", 12), genesis_time=0, justified_checkpoint=cp, finalized_checkpoint=cp,
                     best_justified_checkpoint=cp, proposer_boost_root=bytes(32), equivocating_indices=set(), blocks=blocks)
    assert sp.get_current_slot(store) == current_slot
    seen = set()
    for w, st in zip(wires, r.status):
        if st not in (0, 9, 10, 11, 12, 13):
            continue
        seen.add(int(st))
        bits = IO._decode(w, 8)[1]
        att = PS.Attestation(bits, IO.data_from_bytes(w[4:132]), w[132:228])
        try:
            sp.validate_on_attestation(store, att, False)
            raised = False
        except (AssertionError, KeyError):
            raised = True
        assert raised == (9 <= st <= 12), st
    return seen


def test_grouping_equals_a_hand_built_vote_form():
    """committee 2 (slot 25, index 0): positions 0 and 2 sign data A, 1 signs B, 3 nothing, and position 0 again with B (a duplicate);
    every other committee keeps nothing and has one placeholder"""
    parent = np.array([0, 0, 1], dtype=np.uint32)
    slot = np.array([20, 23, 25], dtype=np.uint64)
    roots = np.array([[b] * 32 for b in (1, 2, 3)], dtype=np.uint8)
    blocks, ids = IO.block_store(parent, slot, roots)
    off = np.array([0, 0, 0, 4] + [8] * 13, dtype=np.int64)
    A = IO.data128(25, 0, bytes(roots[2]), 2, bytes(roots[0]), 3, bytes(roots[1]))
    B = IO.data128(25, 0, bytes(roots[1]), 2, bytes(roots[0]), 3, bytes(roots[1]))
    sig = [bytes([k + 1]) * 96 for k in range(4)]
    one = lambda p: [j == p for j in range(4)]      # noqa: E731
    wires = [IO.encode(one(1), B, sig[0]), IO.encode(one(0), A, sig[1]), IO.encode(one(2), A, sig[2]), IO.encode(one(0), B, sig[3])]
    r = IO.intake_plain(wires, off, 3, 26, DOMAIN, CPS, SPE, 1, blocks, ids)
    assert r.status.tolist() == [0, 0, 0, 13]
    # committee 2's votes in the order of their smallest position: A (position 0) first, then B (position 1)
    assert r.vote.tolist() == [2, 3, 2, IO.NONE] + [IO.NONE] * 4
    assert r.vote_off.tolist() == [0, 1, 2] + list(range(4, 18))
    assert [bytes(x) for x in r.sigs] == [sig[1], sig[0], sig[2]] + [bytes(96)] * 5
    assert bytes(r.data128[2]) == A and bytes(r.data128[3]) == B
    assert not np.delete(r.data128, [2, 3], axis=0).any() and not np.delete(r.msgs, [2, 3], axis=0).any()
    assert r.block_idx.tolist() == [0, 0, 2, 1] + [0] * 13
    assert r.target_epoch[2:4].tolist() == [3, 3] and r.source_epoch[2:4].tolist() == [2, 2]
    assert bytes(r.msgs[2]) == PS.Spec.compute_signing_root(IO.data_from_bytes(A), DOMAIN)


@pytest.mark.parametrize("seed", range(5))
def test_numpy_form_equals_plain_form(seed):
    epoch = 3
    tree, wires = _epoch(100 + seed, epoch, n_extra=40)
    assert len({len(w) for w in wires}) == 1
    blocks, ids = IO.block_store(*tree)
    args = (_layout(), epoch, (epoch + 1) * SPE + 1, DOMAIN, CPS, SPE, 1)
    a = IO.intake_plain(wires, *args, blocks, ids)
    b = IO.intake_numpy(np.frombuffer(b"".join(wires), dtype=np.uint8).reshape(len(wires), -1), *args, *tree)
    assert set(a.status.tolist()) >= {0, 1, 2, 4, 5, 6, 7, 9, 10, 13}
    for f in ("status", "vote", "vote_off", "sigs", "data128", "msgs", "source_epoch", "target_epoch", "block_idx"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def test_ragged_epoch_has_the_requested_groups_and_late_duplicates():
    """ragged_epoch: the requested number of distinct data per committee, whatever its size; with dup = 1 every attestation has a later
    copy, and where the earlier one was made to fail (status 10) the later one is the position's kept attestation"""
    rng = np.random.default_rng(8)
    sizes, distinct = [1, 2, 9, 64, 64], [1, 2, 3, 64, 5]
    tree = IO.random_tree(rng, 30, 3 * 5 - 7)
    wires = IO.ragged_epoch(rng, 3, 5, 1, sizes, tree, distinct=distinct, dup=1.0)
    r = IO.intake_plain(wires, IO.ragged_layout(sizes), 3, 4 * 5, DOMAIN, 1, 5, 8, *IO.block_store(*tree))
    n = sum(sizes)
    assert len(wires) == 2 * n and (r.status[:n] != 13).all() and (r.vote != IO.NONE).all()
    assert np.diff(r.vote_off).tolist() == distinct
    late = r.status[n:].tolist()
    assert 10 in r.status[:n].tolist() and 0 in late and 13 in late and set(late) <= {0, 13}


def test_ragged_numpy_form_equals_plain_form():
    """committees of one size through ragged_epoch, with 2 048 members and every member's own data in one of them"""
    rng = np.random.default_rng(9)
    tree = IO.random_tree(rng, 30, 0)
    wires = IO.ragged_epoch(rng, 3, 2, 1, [2048, 2048], tree, distinct=[2048, 3], absent=0.1, dup=0.05, corrupt=0.1)
    off = IO.ragged_layout([2048, 2048]).astype(np.int64)
    a = IO.intake_plain(wires, off, 3, 8, DOMAIN, 1, 2, 256, *IO.block_store(*tree))
    b = IO.intake_numpy(np.frombuffer(b"".join(wires), dtype=np.uint8).reshape(len(wires), -1), off, 3, 8, DOMAIN, 1, 2, 256, *tree)
    assert int(a.vote_off[1]) > 1500
    for f in ("status", "vote", "vote_off", "sigs", "data128", "msgs", "source_epoch", "target_epoch", "block_idx"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
