"""GPU parity tests for the fork-choice half (K7-K9): latest-message table, per-block weights and
head index against the numpy oracle (oracle/fast.py), at small sizes and at BASELINE.json's
10 000 blocks / 2^20 validators."""
import numpy as np
import pytest

import scenarios
from oracle import fast

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _registry(eng, n, eff, active):
    """fork choice never touches the pubkeys: load a registry of copies of one valid key."""
    from oracle.bls12_381 import G1, g1_compress
    pk = np.tile(np.frombuffer(g1_compress(G1), dtype=np.uint8), (n, 1))
    eng.registry_load(pk, eff, active)


@pytest.mark.parametrize("n_val,n_blk,seed", [(64, 1, 1), (64, 2, 2), (1000, 50, 3), (5000, 300, 4), (1 << 20, 10000, 4), (3000, 14000, 6), (3000, 20000, 7),
                                              # the edges of every form of the tree phase and the vote scatter (tests/test_gpu_forkchoice_forms.py)
                                              (64, 3, 8), (3000, 1023, 9), (3000, 1024, 10), (3000, 1025, 11), (3000, 11264, 12), (3000, 11265, 13),
                                              (3000, 11570, 14), (3000, 11571, 15), (3000, 14463, 16), (3000, 14464, 17), (3000, 25600, 18),
                                              (3000, 25601, 19), (3000, 32767, 20), (3000, 32768, 21), (3000, 65537, 22)])
def test_weights_and_head(eng, n_val, n_blk, seed):
    parent, slot, roots, leaf_viable = scenarios.fork_tree(n_blk, seed)
    msg_block, has_msg, equiv, active, eff = scenarios.votes(n_val, n_blk, seed)
    _registry(eng, n_val, eff, active)
    eng.tree_load(parent, slot, roots, leaf_viable)
    epoch = np.full(n_val, 3, dtype=np.uint64)
    eng.latest_messages_load(epoch, msg_block, has_msg, equiv)
    boost = fast.proposer_boost_score(eff, active, 32, 40)
    for boost_idx in (-1, n_blk - 1, n_blk // 2):
        w_ref = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, boost_idx, boost)
        w = eng.get_weights(boost_idx, boost)
        assert np.array_equal(w, w_ref)
        keep = fast.ghost_viable(parent, leaf_viable)
        assert eng.get_head(0, boost_idx, boost) == fast.ghost_head(parent, roots, keep, w_ref, 0)
    # a second call must see a clean accumulator
    assert np.array_equal(eng.get_weights(-1, 0), fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, -1, 0))


def test_head_tie_break_by_root(eng):
    """all weights zero: the walk must follow the lexicographically highest root at every fork (ref :1114-1116)."""
    parent, slot, roots, leaf_viable = scenarios.fork_tree(200, 9)
    leaf_viable[:] = 1
    n_val = 128
    eff = np.full(n_val, 32 * 10**9, dtype=np.uint64)
    _registry(eng, n_val, eff, np.ones(n_val, dtype=np.uint8))
    eng.tree_load(parent, slot, roots, leaf_viable)
    eng.latest_messages_reset()
    keep = fast.ghost_viable(parent, leaf_viable)
    w0 = np.zeros(200, dtype=np.uint64)
    assert eng.get_head(0) == fast.ghost_head(parent, roots, keep, w0, 0)
    assert eng.get_head(17) == fast.ghost_head(parent, roots, keep, w0, 17)


def test_latest_messages_update_order_exact(eng):
    rng = np.random.default_rng(12)
    n_val, n_blk, n_agg, csize = 4096, 64, 96, 128
    eff = np.full(n_val, 32 * 10**9, dtype=np.uint64)
    _registry(eng, n_val, eff, np.ones(n_val, dtype=np.uint8))
    msg_epoch = rng.integers(0, 3, size=n_val).astype(np.uint64)
    msg_block = rng.integers(0, n_blk, size=n_val).astype(np.uint32)
    has_msg = (rng.random(n_val) < 0.5).astype(np.uint8)
    equiv = (rng.random(n_val) < 0.05).astype(np.uint8)
    msg_block[has_msg == 0] = 0
    eng.latest_messages_load(msg_epoch, msg_block, has_msg, equiv)
    # overlapping committees on purpose: the same validator appears in several attestations of the batch
    members = rng.integers(0, n_val, size=(n_agg, csize)).astype(np.uint32)
    for a in range(n_agg):
        members[a] = rng.permutation(n_val)[:csize]
    off = np.arange(0, (n_agg + 1) * csize, csize, dtype=np.uint32)
    bits = rng.integers(0, 256, size=(n_agg, csize // 8)).astype(np.uint8)
    target_epoch = rng.integers(0, 5, size=n_agg).astype(np.uint64)
    block_idx = rng.integers(0, n_blk, size=n_agg).astype(np.uint32)
    accept = (rng.random(n_agg) < 0.8).astype(np.uint8)
    for a in range(n_agg):                      # sequential oracle, list order
        if not accept[a]:
            continue
        sel = [int(members[a, j]) for j in range(csize) if (bits[a, j >> 3] >> (j & 7)) & 1]
        fast.lmd_update(msg_epoch, msg_block, has_msg, equiv, sel, int(target_epoch[a]), int(block_idx[a]))
    eng.latest_messages_update(members.reshape(-1), off, bits, target_epoch, block_idx, accept)
    e, b, h = eng.latest_messages_read()
    assert np.array_equal(h, has_msg)
    assert np.array_equal(e[h == 1], msg_epoch[h == 1])
    assert np.array_equal(b[h == 1], msg_block[h == 1])


@pytest.mark.parametrize("n,rounds", [(1, 10), (2, 10), (37, 10), (257, 90), (1000, 90), (1 << 20, 90)])
def test_gpu_shuffle_matches_oracle(eng, n, rounds):
    """compute_shuffled_index for the whole list on the GPU (SHA-256 + swap-or-not) vs the numpy oracle."""
    import hashlib
    seed = hashlib.sha256(b"shuffle" + n.to_bytes(4, "little")).digest()
    ref = fast.shuffle_permutation(n, seed, rounds)
    assert np.array_equal(eng.shuffle_committees(seed, n, rounds), ref)
    active = (np.arange(n, dtype=np.uint32) * 3 + 7).astype(np.uint32)
    assert np.array_equal(eng.shuffle_committees(seed, n, rounds, active), active[ref])


@pytest.mark.parametrize("length", [0, 1, 32, 33, 37, 55, 56, 63, 64, 65, 100, 143])
def test_gpu_sha256_batch(eng, length):
    import hashlib
    rng = np.random.default_rng(length)
    n = 70
    msgs = rng.integers(0, 256, size=(n, length), dtype=np.uint8) if length else n
    out = eng.sha256_batch(msgs, length)
    for i in range(n):
        m = bytes(msgs[i]) if length else b""
        assert bytes(out[i]) == hashlib.sha256(m).digest(), (length, i)


def test_gpu_signing_roots_match_oracle(eng):
    from oracle import spec as OS
    from oracle.ssz import compute_domain
    rng = np.random.default_rng(8)
    n = 300
    datas, doms, ser = [], [], []
    for i in range(n):
        d = OS.AttestationData(int(rng.integers(0, 2**62)), int(rng.integers(0, 64)), bytes(rng.integers(0, 256, 32, dtype=np.uint8)),
                               OS.Checkpoint(int(rng.integers(0, 2**40)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))),
                               OS.Checkpoint(int(rng.integers(0, 2**40)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))))
        dom = compute_domain(OS.DOMAIN_BEACON_ATTESTER, bytes(rng.integers(0, 256, 4, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8)))
        datas.append(d)
        doms.append(dom)
        ser.append(d.slot.to_bytes(8, "little") + d.index.to_bytes(8, "little") + d.beacon_block_root + d.source.epoch.to_bytes(8, "little")
                   + d.source.root + d.target.epoch.to_bytes(8, "little") + d.target.root)
    out = eng.signing_roots(np.frombuffer(b"".join(ser), dtype=np.uint8), np.frombuffer(b"".join(doms), dtype=np.uint8))
    for i in range(n):
        assert bytes(out[i]) == OS.Spec.compute_signing_root(datas[i], doms[i])
    one = eng.signing_roots(np.frombuffer(b"".join(ser), dtype=np.uint8), np.frombuffer(doms[0], dtype=np.uint8))
    for i in range(n):
        assert bytes(one[i]) == OS.Spec.compute_signing_root(datas[i], doms[0])


def test_fork_choice_variants_expiry_slashed_equivocation(eng):
    """SURVEY.md section 8(f)-4: vote expiry (min epoch), v1.3 slashed exclusion, on_attester_slashing marking -- vs numpy."""
    n_val, n_blk = 6000, 400
    parent, slot, roots, leaf_viable = scenarios.fork_tree(n_blk, 11)
    msg_block, has_msg, equiv, active, eff = scenarios.votes(n_val, n_blk, 11)
    rng = np.random.default_rng(11)
    epochs = rng.integers(1, 9, size=n_val).astype(np.uint64)
    slashed = (rng.random(n_val) < 0.05).astype(np.uint8)
    flags = (active | (slashed << 1)).astype(np.uint8)
    _registry(eng, n_val, eff, flags)
    eng.tree_load(parent, slot, roots, leaf_viable)
    eng.latest_messages_load(epochs, msg_block, has_msg, equiv)
    keep = fast.ghost_viable(parent, leaf_viable)
    for min_epoch, excl in ((0, False), (5, False), (0, True), (7, True)):
        eng.set_fork_choice_params(min_epoch, excl)
        hm = has_msg & (epochs >= min_epoch).astype(np.uint8)
        act = active & (1 - slashed) if excl else active
        w_ref = fast.ghost_weights(parent, msg_block, hm, eff, act, equiv, -1, 0)
        assert np.array_equal(eng.get_weights(), w_ref)
        assert eng.get_head(0) == fast.ghost_head(parent, roots, keep, w_ref, 0)
    eng.set_fork_choice_params(0, False)
    a1 = np.unique(rng.integers(0, n_val, size=500)).astype(np.uint32)
    a2 = np.unique(rng.integers(0, n_val, size=500)).astype(np.uint32)
    eng.on_attester_slashing(a1, a2)
    eq2 = equiv.copy()
    eq2[np.intersect1d(a1, a2)] = 1
    assert len(np.intersect1d(a1, a2)) > 0
    w_ref = fast.ghost_weights(parent, msg_block, has_msg, eff, active, eq2, -1, 0)
    assert np.array_equal(eng.get_weights(), w_ref)


def test_attestations_wire_decode_matches_oracle(eng):
    """b2_attestations_decode (SSZ wire form of Attestation, pos-evolution.md:714-717) against the oracle's (de)serialiser:
    every bit length around the byte boundaries up to MAX_VALIDATORS_PER_COMMITTEE, random payloads, and the malformed shapes
    (no delimiter, empty bitlist, too long, wrong offset, truncated)."""
    from oracle import ssz
    rng = np.random.default_rng(9)
    limit, stride = 2048, 256
    lengths = list(range(0, 20)) + [63, 64, 65, 511, 512, 513, 2040, 2047, 2048] + [int(x) for x in rng.integers(1, 2049, size=60)]
    enc, want = [], []
    for n in lengths:
        bits = [bool(b) for b in rng.integers(0, 2, size=n)]
        data, sig = bytes(rng.integers(0, 256, size=128, dtype=np.uint8)), bytes(rng.integers(0, 256, size=96, dtype=np.uint8))
        e = ssz.serialize_attestation(bits, data, sig)
        assert ssz.deserialize_attestation(e, limit) == (bits, data, sig)
        enc.append(e)
        want.append((0, bits, data, sig))
    good = enc[30]
    bad = [(good[:-1] + b"\x00", 2),                                        # last byte zero: no delimiter
           (good[:228], 2),                                                 # empty bitlist
           (ssz.serialize_attestation([True] * 2049, bytes(128), bytes(96)), 3),   # one bit over the limit
           (b"\xe5" + good[1:], 1),                                         # wrong offset
           (good[:100], 1),                                                 # truncated container
           (b"", 1)]
    for e, code in bad:
        try:
            ssz.deserialize_attestation(e, limit)
            raise AssertionError("oracle accepted a malformed encoding")
        except ValueError:
            pass
        enc.append(e)
        want.append((code, [], bytes(128), bytes(96)))
    off = np.zeros(len(enc) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(e) for e in enc])
    bits, blen, data, sig, st = eng.attestations_decode(b"".join(enc), off, stride, limit)
    for a, (code, wbits, wdata, wsig) in enumerate(want):
        assert int(st[a]) == code, a
        assert int(blen[a]) == len(wbits), a
        row = np.unpackbits(bits[a], bitorder="little")
        assert [bool(x) for x in row[:len(wbits)]] == wbits and not row[len(wbits):].any(), a
        assert data[a].tobytes() == wdata and sig[a].tobytes() == wsig, a


@pytest.mark.parametrize("n_val,n_blk,seed", [(5000, 300, 4), (1 << 20, 10000, 4), (70000, 14000, 6)])
def test_get_head_forms_agree(eng, n_val, n_blk, seed):
    """The forms of get_head give the oracle's head: the one-launch kernel (b2_get_head, default), the two-launch form (a context
    created with B2_HEAD_FUSED=0), the NVLink-fused multi-rank kernel on a box of one rank (b2_get_head_multi, world = 1: scatter,
    push into its own accumulator, flag exchange with itself, tree), also when only a validator range is scattered; repeated calls
    (double-buffered accumulators, sequence numbers) stay correct; justified roots other than block 0 and the boost are honoured."""
    import os
    from pos_evolution_b200.engine import Engine
    parent, slot, roots, leaf_viable = scenarios.fork_tree(n_blk, seed)
    msg_block, has_msg, equiv, active, eff = scenarios.votes(n_val, n_blk, seed)
    keep = fast.ghost_viable(parent, leaf_viable)
    boost = fast.proposer_boost_score(eff, active, 32, 40)
    os.environ["B2_HEAD_FUSED"] = "0"
    try:
        eng2 = Engine(0)
    finally:
        del os.environ["B2_HEAD_FUSED"]
    for e in (eng, eng2):
        _registry(e, n_val, eff, active)
        e.tree_load(parent, slot, roots, leaf_viable)
        e.latest_messages_load(np.full(n_val, 3, dtype=np.uint64), msg_block, has_msg, equiv)
    eng.fc_exchange_setup(0, 1)
    for justified, boost_idx in ((0, -1), (0, n_blk - 1), (n_blk // 3, n_blk // 2), (0, -1)):
        w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, boost_idx, boost)
        want = fast.ghost_head(parent, roots, keep, w, justified)
        for rep in range(3):
            assert eng.get_head(justified, boost_idx, boost) == want
            assert eng2.get_head(justified, boost_idx, boost) == want
            assert eng.get_head_multi(0, n_val, justified, boost_idx, boost) == want
    # a validator range only: the head of the sub-population
    lo, hi = n_val // 4, n_val // 2
    sub = np.zeros(n_val, dtype=np.uint8)
    sub[lo:hi] = has_msg[lo:hi]
    w = fast.ghost_weights(parent, msg_block, sub, eff, active, equiv, -1, 0)
    assert eng.get_head_multi(lo, hi, 0, -1, 0) == fast.ghost_head(parent, roots, keep, w, 0)
    assert eng.get_head(0, -1, 0) == fast.ghost_head(parent, roots, keep, fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, -1, 0), 0)
    eng2.close()
