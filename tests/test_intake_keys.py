"""tests/intake_keys.py on the CPU: the per-lane inverse, the collision and root-set builders, the restated fingerprint pinned to the
kernels' source text, and the two intake oracles grouping colliding AttestationData by their bytes."""
import os
import re

import numpy as np
import pytest

import aggregate_intake_oracle as AO
import intake_keys as K
import intake_oracle as IO

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pos_evolution_b200", "csrc")


def test_unlane_inverts_every_lane():
    rng = np.random.default_rng(1)
    for k in range(32):
        for w in [0, 1, K.M32, 0x80000000] + rng.integers(0, 1 << 32, 200, dtype=np.uint64).tolist():
            assert K.unlane(K.lane(int(w), k), k) == w
            assert K.lane(K.unlane(int(w), k), k) == w


def test_fingerprint_is_xor_of_lanes():
    d = bytes(range(128))
    want = 0
    for k in range(32):
        w = int.from_bytes(d[4 * k:4 * k + 4], "little")
        x = ((w ^ (k * 0x9E3779B9 & K.M32)) * 0x85EBCA6B) & K.M32
        want ^= x ^ (x >> 15)
    assert K.fingerprint(d) == want


@pytest.mark.parametrize("name,word_load", [("intake.cuh", "w + 4 + 4 * lane"), ("aggintake.cuh", "d + 4 * lane")])
def test_fingerprint_matches_the_kernels(name, word_load):
    """The device fingerprint, as tests/intake_keys.py restates it.  If this fails, the kernel's fingerprint changed: update
    tests/intake_keys.py (lane, unlane, fingerprint), or the collision tests of test_gpu_intake_keys.py silently stop colliding."""
    src = open(os.path.join(CSRC, name)).read()
    lines = [ln.strip() for ln in src.splitlines()]
    i = next(j for j, ln in enumerate(lines) if re.search(r"const uint8_t\* dw = " + re.escape(word_load) + ";", ln))
    block = " ".join(lines[i:i + 4])
    assert "(uint32_t)dw[0] | (uint32_t)dw[1] << 8 | (uint32_t)dw[2] << 16 | (uint32_t)dw[3] << 24) ^ (lane * 0x9e3779b9u)" in block, block
    assert "x *= 0x85ebca6bu;" in block, block
    assert "h = __reduce_xor_sync(B2_FULL_MASK, x ^ (x >> 15));" in block, block
    assert (K.LANE_KEY, K.MIX) == (0x9E3779B9, 0x85EBCA6B)


def test_collisions_collide():
    rng = np.random.default_rng(2)
    d = rng.integers(0, 256, 128, dtype=np.uint8).tobytes()
    for change, fix in ((14, 15), (4, 15), (31, 20), (12, 21)):
        e = K.collide(d, change, fix)
        assert e != d and K.fingerprint(e) == K.fingerprint(d)
        assert e[:4 * min(change, fix)] == d[:4 * min(change, fix)]
    for target in (0, 1, K.M32, 0x12345678):
        for fix in K.FREE_LANES:
            assert K.fingerprint(K.with_fingerprint(d, target, fix)) == target
    s = K.source_lane_set(d, 257)
    assert len(set(s)) == 257 and len({K.fingerprint(x) for x in s}) == 1
    assert all(x[:56] == d[:56] and x[64:] == d[64:] for x in s)      # only the source root's first two words differ


def test_root_builders():
    rng = np.random.default_rng(3)
    groups = K.shared_prefix_groups(rng)
    assert sorted(groups) == list(K.PREFIX_BYTES)
    for p, g in groups.items():
        assert g == sorted(g) and all(r[:p] == g[0][:p] and r[p + 1:] == g[0][p + 1:] for r in g)
    for a, b in K.le_flip_pairs(rng):
        assert b < a and K.le_word_less(a, b)
    lo, hi = K.edge_roots()
    assert lo == bytes(32) and hi < K.OUTSIDE
    r = groups[16][0]
    nm = K.near_misses(r, [r])
    assert len(nm) == 64 and all(sum(x != y for x, y in zip(m, r)) == 1 for m in nm)
    assert K.near_misses(hi, [hi]).count(K.OUTSIDE) == 0


# ------------------------------------------------------------------------------------------ the oracles group by bytes
EPOCH, SPE = 3, 4
PARENT = np.array([0, 0, 1], np.uint32)
SLOT = np.array([10, 12, 13], np.uint64)
ROOTS = np.array([[0x10 + b] * 32 for b in range(3)], np.uint8)


def _x():
    return IO.data128(14, 0, bytes(ROOTS[2]), 2, bytes(32), EPOCH, bytes(ROOTS[1]))


def test_intake_oracles_keep_colliding_data_apart():
    x = _x()
    x2 = K.collide(x, 14, 15)
    off = IO.ragged_layout([2, 2, 4, 2])
    wires = [IO.encode([j == p for j in range(4)], d, bytes([p]) * 96) for p, d in enumerate([x, x2, x, x2])]
    blocks, ids = IO.block_store(PARENT, SLOT, ROOTS)
    r = IO.intake_plain(wires, off, EPOCH, 16, bytes(32), 1, SPE, 1, blocks, ids)
    assert r.status.tolist() == [0, 0, 0, 0]
    assert r.vote[4:8].tolist() == [2, 3, 2, 3] and r.vote_off.tolist() == [0, 1, 2, 4, 5]
    assert bytes(r.data128[2]) == x and bytes(r.data128[3]) == x2 and bytes(r.msgs[2]) != bytes(r.msgs[3])
    rec = np.frombuffer(b"".join(wires), np.uint8).reshape(4, -1)
    n = IO.intake_numpy(rec, off.astype(np.int64), EPOCH, 16, bytes(32), 1, SPE, 1, PARENT, SLOT, ROOTS)
    for f in ("status", "vote", "vote_off", "sigs", "data128", "msgs", "block_idx"):
        assert np.array_equal(getattr(n, f), getattr(r, f)), f


def test_aggregate_oracle_keeps_colliding_data_apart():
    """accepted A (X, bits S); B (colliding X', bits in S) is accepted; C (X, bits in S) is check 10; D (X', bits in B's) is check 10"""
    x = _x()
    x2 = K.collide(x, 14, 15)
    members = np.arange(8, dtype=np.uint32)
    off = np.array([0, 2, 2, 6, 8], np.uint32)                      # committee 2 (slot 14, index 0) = members 2..5
    items = [(2, [1, 1, 1, 0], x), (3, [1, 1, 0, 0], x2), (4, [0, 1, 0, 0], x), (5, [1, 0, 0, 0], x2)]
    wires = [AO.encode(a, b, d, bytes(96), bytes([a]) * 96, bytes(96)) for a, b, d in items]
    r = AO.validate(wires, members, off, EPOCH, 14, bytes(96), 1, SPE, 1, PARENT, SLOT, ROOTS, lambda i: (True, True, True), 16, 32)
    assert r.status.tolist() == [0, 0, 10, 10]
    assert r.data_id.tolist() == [0, 1, 0, 1]
