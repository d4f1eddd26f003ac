"""The error contract of the C ABI (include/b200pos.h): on error no output buffer and no device table is modified.

Each synchronous entry point gets one argument its host check rejects, with output arrays the test owns and fills with a sentinel
byte.  The call must return B2_EINVAL, leave every output byte as it was, and leave the device tables answering as before.  A
registry load that fails on the device (out of memory) must keep the previous registry and leave the next calls unaffected."""
import ctypes

import numpy as np
import pytest

import scenarios

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
N_VAL, N_BLK, N_AGG, CSIZE = 256, 40, 4, 8


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _sentinel(*shape_dtypes):
    return [np.full(shape, SENTINEL, dtype=np.uint8).view(dtype) for shape, dtype in shape_dtypes]


def _batch(rng, n_val):
    members = rng.integers(0, n_val, size=N_AGG * CSIZE).astype(np.uint32)
    off = np.arange(0, (N_AGG + 1) * CSIZE, CSIZE, dtype=np.uint32)
    bits = np.full((N_AGG, CSIZE // 8), 0xFF, dtype=np.uint8)
    return members, off, bits


def _load_state(eng, n_val, seed):
    """registry of distinct keys, a fork tree, latest messages and both participation tables"""
    rng = np.random.default_rng(seed)
    eff = rng.integers(16, 33, size=n_val).astype(np.uint64) * np.uint64(10**9)
    assert eng.registry_load(eng.sk_to_pk(list(range(1, n_val + 1))), eff).all()
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, seed)
    eng.tree_load(parent, slot, roots, leaf_viable)
    has_msg = (rng.random(n_val) < 0.8).astype(np.uint8)
    eng.latest_messages_load(rng.integers(0, 9, size=n_val).astype(np.uint64), rng.integers(0, N_BLK, size=n_val).astype(np.uint32), has_msg,
                             (rng.random(n_val) < 0.05).astype(np.uint8))
    for which in (0, 1):
        eng.participation_load(which, rng.integers(0, 8, size=n_val).astype(np.uint8))


def _device_state(eng):
    return [*eng.latest_messages_read(), eng.participation_read(0), eng.participation_read(1), eng.get_weights(), eng.get_head(0)]


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    _load_state(e, N_VAL, 3)
    yield e
    e.close()


def _g1_aggregate(lib, h, rng):
    members, off, bits = _batch(rng, N_VAL)
    members[5] = N_VAL
    out = _sentinel(((N_AGG, 48), np.uint8), (N_AGG, np.uint8))
    return lib.b2_g1_aggregate(h, _p(members), _p(off), _p(bits), bits.shape[1], N_AGG, *map(_p, out)), out, "outside the registry"


def _aggregate(lib, h, rng):
    sigs = np.zeros((4, 96), dtype=np.uint8)
    seg_off = np.array([0, 3, 2, 4], dtype=np.uint32)
    out = _sentinel(((3, 96), np.uint8), (3 * 4, np.int32))
    return lib.b2_aggregate(h, _p(sigs), _p(seg_off), 3, *map(_p, out)), out, "seg_off"


def _fast_aggregate_verify(lib, h, rng):
    members, off, bits = _batch(rng, N_VAL)
    off = off + np.uint32(1)
    msgs, sigs = np.zeros((N_AGG, 32), dtype=np.uint8), np.zeros((N_AGG, 96), dtype=np.uint8)
    out = _sentinel((N_AGG, np.uint8))
    return lib.b2_fast_aggregate_verify(h, _p(members), _p(off), _p(bits), bits.shape[1], _p(msgs), _p(sigs), N_AGG, _p(out[0])), out, "off"


def _fast_aggregate_verify_pks(lib, h, rng):
    pks = np.zeros((6, 48), dtype=np.uint8)
    pk_off = np.array([0, 2, 1, 6], dtype=np.uint32)
    msgs, sigs = np.zeros((3, 32), dtype=np.uint8), np.zeros((3, 96), dtype=np.uint8)
    out = _sentinel((3, np.uint8))
    return lib.b2_fast_aggregate_verify_pks(h, _p(pks), _p(pk_off), _p(msgs), _p(sigs), 3, _p(out[0])), out, "pk_off"


def _sign(lib, h, rng):
    sk8 = np.ones((3, 8), dtype=np.uint32)
    msg_idx = np.array([0, 2, 1], dtype=np.uint32)
    msgs = np.zeros((2, 32), dtype=np.uint8)
    out = _sentinel(((3, 96), np.uint8))
    return lib.b2_sign(h, _p(sk8), _p(msg_idx), 3, _p(msgs), 2, _p(out[0])), out, "msg_idx"


def _attestations_decode(lib, h, rng):
    n, stride = 3, 8
    wire = np.zeros(700, dtype=np.uint8)
    woff = np.array([0, 300, 200, 700], dtype=np.uint32)
    out = _sentinel(((n, stride), np.uint8), (n * 4, np.uint32), ((n, 128), np.uint8), ((n, 96), np.uint8), (n * 4, np.int32))
    return lib.b2_attestations_decode(h, _p(wire), _p(woff), n, stride, 64, *map(_p, out)), out, "woff"


def _latest_messages_load(lib, h, rng):
    epoch = np.full(N_VAL, 5, dtype=np.uint64)
    epoch[7] = 0xFFFFFFFF
    block, has_msg, equiv = np.zeros(N_VAL, dtype=np.uint32), np.ones(N_VAL, dtype=np.uint8), np.zeros(N_VAL, dtype=np.uint8)
    return lib.b2_latest_messages_load(h, _p(epoch), _p(block), _p(has_msg), _p(equiv), N_VAL), [], "32 bits"


def _latest_messages_update(lib, h, rng):
    members, off, bits = _batch(rng, N_VAL)
    target = np.full(N_AGG, 7, dtype=np.uint64)
    target[1] = 0xFFFFFFFF
    block, accept = np.ones(N_AGG, dtype=np.uint32), np.ones(N_AGG, dtype=np.uint8)
    return (lib.b2_latest_messages_update(h, _p(members), _p(off), _p(bits), bits.shape[1], _p(target), _p(block), _p(accept), N_AGG), [],
            "32 bits")


def _participation_update(lib, h, rng):
    members, off, bits = _batch(rng, N_VAL)
    members[-1] = N_VAL + 1000
    mask, accept = np.full(N_AGG, 7, dtype=np.uint8), np.ones(N_AGG, dtype=np.uint8)
    out = _sentinel((N_AGG * 8, np.uint64))
    return (lib.b2_participation_update(h, 0, _p(members), _p(off), _p(bits), bits.shape[1], _p(mask), _p(accept), N_AGG, 10**9, 7777, _p(out[0])),
            out, "outside the registry")


def _on_attester_slashing(lib, h, rng):
    i1 = np.array([1, 5, 3, 9], dtype=np.uint32)
    i2 = np.array([1, 3, 5, 9], dtype=np.uint32)
    return lib.b2_on_attester_slashing(h, _p(i1), 4, _p(i2), 4), [], "sorted"


def _tree_load(lib, h, rng):
    parent, slot, roots, viable = scenarios.fork_tree(N_BLK + 10, 11)
    parent[N_BLK] = N_BLK
    return lib.b2_tree_load(h, _p(parent), _p(slot), _p(roots), _p(viable), N_BLK + 10), [], "topological"


def _get_head(lib, h, rng):
    out = _sentinel((4, np.uint32))
    return lib.b2_get_head(h, N_BLK, -1, 0, _p(out[0])), out, "out of range"


CASES = {f.__name__[1:]: f for f in (_g1_aggregate, _aggregate, _fast_aggregate_verify, _fast_aggregate_verify_pks, _sign, _attestations_decode,
                                     _latest_messages_load, _latest_messages_update, _participation_update, _on_attester_slashing, _tree_load,
                                     _get_head)}


@pytest.mark.parametrize("entry", list(CASES))
def test_rejected_call_changes_nothing(eng, entry):
    from pos_evolution_b200._lib import B2_EINVAL
    before = _device_state(eng)
    rc, outputs, why = CASES[entry](eng.lib, eng.h, np.random.default_rng(5))
    assert rc == B2_EINVAL
    assert why in eng.lib.b2_last_error(eng.h).decode()
    for o in outputs:
        assert (o.view(np.uint8) == SENTINEL).all()
    after = _device_state(eng)
    for a, b in zip(before, after):
        assert np.array_equal(a, b)


def test_failed_registry_load_keeps_the_old_registry():
    """n = 2^32 - 1: the records table (96 B per validator, allocated before any host array is read) cannot fit, so the load fails
    with cudaErrorMemoryAllocation; the previous tables, and the next launches, must be unaffected."""
    import torch
    from pos_evolution_b200._lib import B2_ECUDA
    from pos_evolution_b200.engine import Engine
    n_bad = (1 << 32) - 1
    if torch.cuda.get_device_properties(0).total_memory >= 96 * n_bad:
        pytest.skip("the device could hold the records table of 2^32 - 1 validators")
    n_val = 4096
    eng = Engine(0)
    _load_state(eng, n_val, 7)
    members, off, bits = _batch(np.random.default_rng(8), n_val)
    agg = eng.g1_aggregate(members, off, bits)
    lmd = eng.latest_messages_read()
    head = eng.get_head(0)
    small = np.zeros(64, dtype=np.uint8)
    assert eng.lib.b2_registry_load(eng.h, _p(small), _p(small), _p(small), n_bad, None) == B2_ECUDA
    for a, b in zip(eng.g1_aggregate(members, off, bits), agg):
        assert np.array_equal(a, b)
    for a, b in zip(eng.latest_messages_read(), lmd):
        assert np.array_equal(a, b)
    assert eng.get_head(0) == head
    eng.close()
