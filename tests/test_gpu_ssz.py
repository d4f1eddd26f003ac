"""hash_tree_root on the GPU (csrc/ssz.cuh through b2_ssz_*) against the hashlib oracle of tests/ssz_oracle.py: chunk roots of basic lists
and vectors, the device validators tree after loads and incremental updates, the error contract, 2^20 and 2^17 validators, and
Spec.hash_tree_root_state on a minimal-preset state before and after mutations."""
import ctypes
import hashlib

import numpy as np
import pytest

import ssz_oracle as O
from pos_evolution_b200 import spec as PS

pytestmark = pytest.mark.gpu

REG_LIMIT = 2**40


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _records(rng, n):
    """n random 121-byte Validator records whose slashed byte is 0 or 1"""
    rec = rng.integers(0, 256, size=(n, 121), dtype=np.uint8)
    rec[:, 88] &= 1
    return rec


def _validator(r) -> PS.Validator:
    u = lambda o: int.from_bytes(bytes(r[o:o + 8]), "little")      # noqa: E731
    return PS.Validator(bytes(r[0:48]), u(80), bool(r[88]), u(97), u(105), withdrawal_credentials=bytes(r[48:80]),
                        activation_eligibility_epoch=u(89), withdrawable_epoch=u(113))


def _oracle_validators_root(rec) -> bytes:
    return O.records_root([bytes(r) for r in rec], REG_LIMIT)


LENGTHS = sorted({0, 1, 2, 3, 31, 32, 33} | {(1 << k) + d for k in (6, 10, 14) for d in (-1, 1)})


@pytest.mark.parametrize("size,dtype", [(1, np.uint8), (8, "<u8"), (32, np.uint8)])
def test_chunks_root_lists_and_vectors(eng, size, dtype):
    """basic lists at the registry limit (uint8 and uint64), lists of roots at HISTORICAL_ROOTS_LIMIT, and the same bytes as vectors"""
    rng = np.random.default_rng(size)
    limit = REG_LIMIT if size < 32 else PS.MAINNET.HISTORICAL_ROOTS_LIMIT
    depth = PS._chunk_depth(limit, size)
    for n in LENGTHS:
        if size == 32:
            vals = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
            want_list = O.roots_list_root([bytes(v) for v in vals], limit)
        else:
            vals = rng.integers(0, 2**63, size=n, dtype=np.uint64).astype(dtype) if size == 8 else rng.integers(0, 256, size=n, dtype=np.uint8)
            want_list = O.basic_list_root([int(v) for v in vals], size, limit)
        assert eng.ssz_chunks_root(vals, depth, n) == want_list, n
        if n:
            want_vec = O.roots_vector_root([bytes(v) for v in vals]) if size == 32 else O.basic_vector_root([int(v) for v in vals], size)
            assert eng.ssz_chunks_root(vals, PS._chunk_depth(n, size)) == want_vec, n


def test_chunks_root_limits(eng):
    """a tree exactly at its limit, and one chunk more than the limit (B2_EINVAL)"""
    from pos_evolution_b200._lib import B2Error, B2_EINVAL
    roots = np.arange(64 * 32, dtype=np.uint32).astype(np.uint8).reshape(64, 32)
    assert eng.ssz_chunks_root(roots, 6, 64) == O.roots_list_root([bytes(r) for r in roots], 64)
    with pytest.raises(B2Error) as e:
        eng.ssz_chunks_root(np.zeros((65, 32), dtype=np.uint8), 6, 65)
    assert e.value.code == B2_EINVAL


@pytest.mark.parametrize("n", [0, 1, 2, 3, 1000, 2**16 + 3])
def test_validators_load(eng, n):
    rec = _records(np.random.default_rng(n), n)
    assert eng.ssz_validators_load(rec) == _oracle_validators_root(rec)


def test_incremental_updates(eng):
    """after each batch (one record, a few, every record, none) the root equals a fresh load of the same records and the oracle"""
    from pos_evolution_b200.engine import Engine
    rng = np.random.default_rng(11)
    n = 5000
    rec = _records(rng, n)
    eng.ssz_validators_load(rec)
    fresh = Engine(0)
    try:
        for k in (1, 7, 64, 1, n, 300, 0, 2):
            idx = np.sort(rng.choice(n, size=k, replace=False)).astype(np.uint32)
            if k == 2:
                idx = np.array([n - 2, n - 1], dtype=np.uint32)       # the last leaves, whose right neighbours are zero leaves
            rec[idx] = _records(rng, k)
            root = eng.ssz_validators_update(idx, rec[idx])
            assert root == fresh.ssz_validators_load(rec), k
            assert root == _oracle_validators_root(rec), k
    finally:
        fresh.close()


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("bad", ["unsorted", "duplicate", "out_of_range"])
def test_rejected_update_changes_nothing(eng, bad):
    from pos_evolution_b200._lib import B2_EINVAL
    rng = np.random.default_rng(21)
    n = 200
    rec = _records(rng, n)
    root = eng.ssz_validators_load(rec)
    idx = {"unsorted": [3, 9, 5], "duplicate": [3, 5, 5], "out_of_range": [3, 9, n]}[bad]
    idx = np.array(idx, dtype=np.uint32)
    new = _records(rng, 3)
    out = np.full(32, 0xA5, dtype=np.uint8)
    assert eng.lib.b2_ssz_validators_update(eng.h, _p(idx), _p(new), 3, _p(out)) == B2_EINVAL
    assert "strictly increasing" in eng.lib.b2_last_error(eng.h).decode()
    assert (out == 0xA5).all()
    assert eng.ssz_validators_update(np.zeros(0, dtype=np.uint32), np.zeros((0, 121), dtype=np.uint8)) == root
    # and the tree still updates correctly afterwards
    rec[[4, 150]] = _records(rng, 2)
    assert eng.ssz_validators_update([4, 150], rec[[4, 150]]) == _oracle_validators_root(rec)


def test_update_without_tree_is_rejected():
    from pos_evolution_b200._lib import B2_EINVAL
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    try:
        out = np.full(32, 0xA5, dtype=np.uint8)
        idx, rec = np.zeros(1, dtype=np.uint32), np.zeros((1, 121), dtype=np.uint8)
        assert e.lib.b2_ssz_validators_update(e.h, _p(idx), _p(rec), 1, _p(out)) == B2_EINVAL
        assert (out == 0xA5).all()
        assert e.launch_count == 0
    finally:
        e.close()


def test_full_size_planted_records(eng):
    """2^20 equal records except k planted ones; the oracle memoises equal subtrees (O(k * 40) hashes).  Then an update of other
    planted records, checked the same way."""
    n, k = 2**20, 50
    rng = np.random.default_rng(31)
    base = _records(rng, 1)[0]
    rec = np.tile(base, (n, 1))
    planted = np.sort(rng.choice(n, size=k, replace=False))
    rec[planted] = _records(rng, k)
    dflt = O.validator_root(_validator(base))
    assert dflt == O.record_root(bytes(base))
    over = {int(i): O.validator_root(_validator(rec[i])) for i in planted}
    assert eng.ssz_validators_load(rec) == O.sparse_list_root(n, dflt, over, REG_LIMIT)
    idx = np.sort(rng.choice(n, size=k, replace=False)).astype(np.uint32)
    rec[idx] = _records(rng, k)
    over.update({int(i): O.validator_root(_validator(rec[i])) for i in idx})
    assert eng.ssz_validators_update(idx, rec[idx]) == O.sparse_list_root(n, dflt, over, REG_LIMIT)


def test_random_records_2_17(eng):
    rec = _records(np.random.default_rng(41), 2**17)
    assert eng.ssz_validators_load(rec) == _oracle_validators_root(rec)


def _minimal_state():
    """a MINIMAL-preset state with every field set (the keys are random bytes: the root only hashes them)"""
    p, n = PS.MINIMAL, 64
    rng = np.random.default_rng(5)
    h = lambda s: hashlib.sha256(s).digest()      # noqa: E731
    validators = [PS.Validator(rng.bytes(48), int(rng.choice([32, 31, 16])) * 10**9, i % 7 == 0, i % 4, PS.FAR_FUTURE_EPOCH if i % 3 else 40 + i,
                               withdrawal_credentials=h(b"wc%d" % i), activation_eligibility_epoch=i % 3,
                               withdrawable_epoch=256 + i if i % 5 == 0 else PS.FAR_FUTURE_EPOCH) for i in range(n)]
    state = PS.BeaconState(
        slot=77, fork=PS.Fork(bytes(4), bytes.fromhex("02000000"), 3), genesis_validators_root=h(b"gvr"), validators=validators,
        balances=[int(x) for x in rng.integers(16 * 10**9, 33 * 10**9, size=n)],
        randao_mixes=[h(b"mix%d" % i) for i in range(p.EPOCHS_PER_HISTORICAL_VECTOR)],
        block_roots=[h(b"block%d" % i) for i in range(p.SLOTS_PER_HISTORICAL_ROOT)],
        previous_epoch_participation=[int(x) for x in rng.integers(0, 8, size=n)], current_epoch_participation=[int(x) for x in rng.integers(0, 8, size=n)],
        previous_justified_checkpoint=PS.Checkpoint(7, h(b"pj")), current_justified_checkpoint=PS.Checkpoint(8, h(b"cj")),
        finalized_checkpoint=PS.Checkpoint(6, h(b"fin")),
        current_sync_committee=PS.SyncCommittee([rng.bytes(48) for _ in range(p.SYNC_COMMITTEE_SIZE)], rng.bytes(48)),
        next_sync_committee=PS.SyncCommittee([rng.bytes(48) for _ in range(p.SYNC_COMMITTEE_SIZE)], rng.bytes(48)))
    state.genesis_time = 1606824023
    state.latest_block_header = PS.BeaconBlockHeader(23, 7, h(b"parent"), h(b"sr"), h(b"body"))
    state.state_roots = [h(b"state%d" % i) for i in range(p.SLOTS_PER_HISTORICAL_ROOT)]
    state.historical_roots = [h(b"hist%d" % i) for i in range(5)]
    state.eth1_data = PS.Eth1Data(h(b"dep"), 64, h(b"eth1"))
    state.eth1_data_votes = [PS.Eth1Data(h(b"v%d" % i), i, h(b"b%d" % i)) for i in range(3)]
    state.eth1_deposit_index = 64
    state.slashings = [int(x) for x in rng.integers(0, 2**40, size=p.EPOCHS_PER_SLASHINGS_VECTOR)]
    state.inactivity_scores = [int(x) for x in rng.integers(0, 100, size=len(state.validators))]
    state.justification_bits = [1, 0, 1, 1]
    state.latest_execution_payload_header = PS.ExecutionPayloadHeader(h(b"ph"), bytes(range(20)), h(b"esr"), h(b"rr"), bytes(range(256)),
                                                                       h(b"rand"), 99, 30_000_000, 12_345, 1_700_000_000, b"graffiti",
                                                                       7 * 10**9, h(b"bh"), h(b"tx"))
    return state


def test_hash_tree_root_state(eng):
    p = PS.MINIMAL
    sp = PS.Spec(p, eng)
    state = _minimal_state()
    assert sp.hash_tree_root_state(state) == O.state_root(state, p)
    # mutate balances, one validator and both participation lists
    state.balances[3] += 10**9
    state.validators[17].effective_balance -= 10**9
    state.validators[17].slashed = True
    state.previous_epoch_participation[0] = 7
    state.current_epoch_participation = [x ^ 1 for x in state.current_epoch_participation]
    assert sp.hash_tree_root_state(state) == O.state_root(state, p)
    state.validators[0].exit_epoch = 9
    state.validators[63].withdrawal_credentials = bytes(32)
    assert sp.hash_tree_root_state(state) == O.state_root(state, p)
    assert sp.stats["ssz_validator_loads"] == 1 and sp.stats["ssz_validator_updates"] == 2
    # defaults: None vectors and sync committees hash as their zero value
    state.state_roots, state.slashings, state.current_sync_committee = None, None, None
    assert sp.hash_tree_root_state(state) == O.state_root(state, p)
    # a grown registry is re-loaded
    state.validators.append(PS.Validator(bytes(48), 32 * 10**9))
    state.balances.append(32 * 10**9)
    assert sp.hash_tree_root_state(state) == O.state_root(state, p)
    assert sp.stats["ssz_validator_loads"] == 2
