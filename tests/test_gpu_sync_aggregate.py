"""Sync-committee aggregates on the GPU (b2_sync_committee_load, b2_sync_aggregate_verify / _dev; kernels in csrc/syncagg.cuh):
the aggregate key byte for byte against b2_aggregate_pks on both sides of the participant / complement switch, adversarial committees
(duplicate keys, P and -P, invalid keys at participating and non-participating positions), the empty-participation rule, two committees
in one call, oracle parity on the minimal preset (verdicts and process_sync_aggregate balances), agreement with FastAggregateVerify
over registry indices at mainnet size (also in RLC mode and through _dev), the error contract, the device guard and the bls facade.
Run on an H100:
    python -m pytest tests/test_gpu_sync_aggregate.py -m gpu"""
import copy
import ctypes

import numpy as np
import pytest

import bls_cases as bc
import sync_oracle as SO
from oracle.bls12_381 import R

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
INF1, INF2 = bc.INF1, bc.INF2


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _rows(bits_list, size):
    """list of 0/1 lists -> uint8[n, ceil(size / 8)] Bitvector rows"""
    out = np.zeros((len(bits_list), (size + 7) // 8), dtype=np.uint8)
    for i, b in enumerate(bits_list):
        if len(b):
            packed = np.packbits(np.asarray(b, dtype=np.uint8), bitorder="little")
            out[i, :packed.shape[0]] = packed
    return out


def _u8(chunks, width):
    return np.frombuffer(b"".join(chunks), dtype=np.uint8).reshape(-1, width)


def _dev_verify(e, cidx, rows, msgs, sigs, want_pk=False):
    import torch
    dev = torch.device("cuda", 0)
    t = [torch.as_tensor(np.array(x), device=dev) for x in (np.asarray(cidx, dtype=np.uint32).astype(np.int32), rows, msgs, sigs)]
    n = len(cidx)
    ok = torch.full((n,), 7, dtype=torch.uint8, device=dev)
    pk = torch.zeros((n, 48), dtype=torch.uint8, device=dev) if want_pk else None
    e.sync_aggregate_verify_dev(t[0], t[1], t[2], t[3], ok, pk)
    torch.cuda.synchronize()
    return ok.cpu().numpy().tolist(), (pk.cpu().numpy() if want_pk else None)


# ------------------------------------------------------------------------------------------ honest committees signed on the GPU
def _committee(e, size, first_sk):
    sks = [first_sk + i for i in range(size)]
    return sks, e.sk_to_pk(sks)


def _sign_blocks(e, sks, bits_list, msgs):
    """honest aggregate signature per block from the summed secret keys of its participants (multiplicity kept); INF2 when none"""
    sums = [sum(sk for sk, b in zip(sks, bits) if b) % R for bits in bits_list]
    nz = [i for i, s in enumerate(sums) if s]
    out = np.tile(np.frombuffer(INF2, dtype=np.uint8), (len(sums), 1))
    if nz:
        out[nz] = e.sign([sums[i] for i in nz], np.arange(len(nz), dtype=np.uint32), msgs[nz])
    return out


@pytest.mark.parametrize("size", [512, 37])
def test_pk48_matches_aggregate_pks_across_the_switch(eng, size):
    """participation k = 0, 1, size/2, size/2 + 1, size - 1, size (random positions): the key written to pk48_out is b2_aggregate_pks of
    the explicit participant keys, and every honest block verifies (the empty one with the infinity signature)"""
    sks, pks = _committee(eng, size, 5000)
    assert eng.sync_committee_load(pks, size).all()
    rng = np.random.default_rng(size)
    ks = [0, 1, size // 2, size // 2 + 1, size - 1, size] * 2
    bits_list = []
    for k in ks:
        b = np.zeros(size, dtype=np.uint8)
        b[rng.permutation(size)[:k]] = 1
        bits_list.append(b.tolist())
    msgs = rng.integers(0, 256, size=(len(ks), 32), dtype=np.uint8)
    sigs = _sign_blocks(eng, sks, bits_list, msgs)
    ok, pk = eng.sync_aggregate_verify(np.zeros(len(ks), dtype=np.uint32), _rows(bits_list, size), msgs, sigs, want_pubkeys=True)
    assert ok.tolist() == [1] * len(ks)
    sel = [pks[np.flatnonzero(b)] for b in bits_list]
    off = np.cumsum([0] + [len(s) for s in sel]).astype(np.uint32)
    want, status = eng.aggregate_pks(np.concatenate(sel), off)
    assert np.array_equal(pk, want)
    assert (status[np.asarray(ks) == 0] == 6).all() and (status[np.asarray(ks) > 0] == 0).all()
    assert bytes(pk[0]) == INF1
    ok_dev, pk_dev = _dev_verify(eng, np.zeros(len(ks), dtype=np.uint32), _rows(bits_list, size), msgs, sigs, want_pk=True)
    assert ok_dev == [1] * len(ks) and np.array_equal(pk_dev, want)


# ------------------------------------------------------------------------------------------ adversarial committees (bls_cases registry)
ADV_SIZE = 16


def _adv_committees():
    """(name, 16 registry names) -- all loaded together, so the blocks below also span four committees of one call"""
    return [("distinct", ["pk%d" % i for i in range(16)]),
            ("duplicates", ["pk5"] * 12 + ["pk6", "pk6", "pk7", "pk5"]),
            ("p_and_neg_p", ["pk3", "neg3"] * 8),
            ("invalid_keys", ["pk8", "enc:not_in_g1", "pk9", "enc:zero_bytes", "pk10", "enc:infinity"] + ["pk%d" % i for i in range(11, 21)])]


def _secret(name):
    if name.startswith("pk"):
        return bc.sk(int(name[2:]))
    if name.startswith("neg"):
        return -bc.sk(int(name[3:]))
    return 0                                                                  # invalid key: no secret behind it


def _adv_blocks():
    """[(committee, bits, signature kind)]: kind "honest" signs with the participants' summed secrets, "inf" is INF2"""
    full, none = [1] * 16, [0] * 16
    nine = [1] * 9 + [0] * 7
    seven = [0] * 9 + [1] * 7
    return [(0, full, "honest"), (0, nine, "honest"), (0, seven, "honest"), (0, none, "inf"), (0, none, "honest_other"),
            (1, full, "honest"), (1, nine, "honest"), (1, seven, "honest"), (1, [1] + [0] * 15, "honest"),
            (1, [1, 1] + [0] * 14, "honest"), (1, [0] * 12 + [1, 1, 0, 0], "honest"),
            (2, full, "inf"), (2, full, "honest"), (2, [1, 1] + [0] * 14, "inf"), (2, [1, 0] * 8, "honest"), (2, [1] * 15 + [0], "honest"),
            (3, full, "honest"), (3, [1, 0, 1, 0, 1, 0] + [1] * 10, "honest"), (3, [1, 0, 1, 0, 1, 0] + [0] * 10, "honest"),
            (3, [0, 1, 0, 0, 0, 0] + [1] * 10, "honest"), (3, [1, 0, 0, 1] + [0] * 12, "honest"), (3, [0] * 5 + [1] + [1] * 10, "honest")]


@pytest.fixture(scope="module")
def adversarial(eng):
    rows, index = bc.registry()
    comms = _adv_committees()
    keys = [rows[index[n]] for _, names in comms for n in names]
    valid = eng.sync_committee_load(_u8(keys, 48), ADV_SIZE)
    with bc.cached_key_validate():
        from oracle import bls_sig as B
        assert valid.tolist() == [int(B.KeyValidate(k)) for k in keys]
    cidx, bits_list, sigs, want, part_keys = [], [], [], [], []
    for c, bits, kind in _adv_blocks():
        names = comms[c][1]
        participants = [n for n, b in zip(names, bits) if b]
        s = sum(_secret(n) for n in participants) % R
        sig = INF2 if kind == "inf" or (kind == "honest" and s == 0) else bc.sign(s if kind == "honest" else bc.sk(99))
        pk = [rows[index[n]] for n in participants]
        with bc.cached_key_validate():
            want.append(int(SO.eth_fast_aggregate_verify(pk, bc.MSG, sig)))
        cidx.append(c)
        bits_list.append(bits)
        sigs.append(sig)
        part_keys.append(pk)
    return np.array(cidx, dtype=np.uint32), _rows(bits_list, ADV_SIZE), np.tile(np.frombuffer(bc.MSG, dtype=np.uint8), (len(cidx), 1)), \
        _u8(sigs, 96), want, part_keys


def test_adversarial_committees(eng, adversarial):
    cidx, rows, msgs, sigs, want, part_keys = adversarial
    blocks = _adv_blocks()
    w = {i: v for i, v in enumerate(want)}
    # the oracle itself: duplicates and the complement side verify; cancellation and invalid participants reject; an invalid key at a
    # non-participating position has no effect; no participants accept exactly the infinity signature
    assert w[0] == w[1] == w[2] == w[3] == 1 and w[4] == 0
    assert all(w[i] == 1 for i in range(5, 11))
    assert w[11] == w[12] == w[13] == 0 and w[14] == w[15] == 1
    assert w[16] == 0 and w[17] == 1 and w[18] == 1 and w[19] == 0 and w[20] == 0 and w[21] == 0
    ok, pk = eng.sync_aggregate_verify(cidx, rows, msgs, sigs, want_pubkeys=True)
    bad = [(i, blocks[i], int(g), x) for i, (g, x) in enumerate(zip(ok, want)) if g != x]
    assert not bad, bad
    off = np.cumsum([0] + [len(k) for k in part_keys]).astype(np.uint32)
    want_pk, _ = eng.aggregate_pks(_u8([k for ks in part_keys for k in ks], 48), off)
    assert np.array_equal(pk, want_pk)
    assert bytes(pk[11]) == bytes(pk[13]) == INF1                             # P and -P cancel
    ok_dev, pk_dev = _dev_verify(eng, cidx, rows, msgs, sigs, want_pk=True)
    assert ok_dev == want and np.array_equal(pk_dev, want_pk)
    eng.set_verify_mode(True, bytes(range(32)))
    try:
        assert eng.sync_aggregate_verify(cidx, rows, msgs, sigs).tolist() == want
    finally:
        eng.set_verify_mode(False)


# ------------------------------------------------------------------------------------------ the empty-participation rule
def test_empty_participation_rule(eng):
    sks, pks = _committee(eng, 32, 7000)
    eng.sync_committee_load(pks, 32)
    honest = _sign_blocks(eng, sks, [[1] * 32], np.zeros((1, 32), dtype=np.uint8))[0].tobytes()
    others = [INF2, honest, bytes(96), INF2[:95] + b"\x01", bytes([0xE0]) + bytes(95), bytes([0x40]) + bytes(95), INF2[:48] + b"\x80" + bytes(47)]
    want = [1] + [0] * (len(others) - 1)
    rows = _rows([[0] * 32] * len(others), 32)
    msgs = np.zeros((len(others), 32), dtype=np.uint8)
    sigs = _u8(others, 96)
    assert eng.sync_aggregate_verify(np.zeros(len(others), dtype=np.uint32), rows, msgs, sigs).tolist() == want
    assert _dev_verify(eng, np.zeros(len(others), dtype=np.uint32), rows, msgs, sigs)[0] == want
    eng.set_verify_mode(True, bytes(range(32)))
    try:
        assert eng.sync_aggregate_verify(np.zeros(len(others), dtype=np.uint32), rows, msgs, sigs).tolist() == want
    finally:
        eng.set_verify_mode(False)
    assert SO.eth_fast_aggregate_verify([], bytes(32), INF2) is True
    assert [SO.eth_fast_aggregate_verify([], bytes(32), s) for s in others] == [bool(x) for x in want]


def test_padding_bits_are_ignored(eng):
    """committee of 37: bits 37..39 of the last byte are not positions"""
    sks, pks = _committee(eng, 37, 8000)
    eng.sync_committee_load(pks, 37)
    bits = [[1] * 37, [0] * 37, [1] * 18 + [0] * 19]
    msgs = np.zeros((3, 32), dtype=np.uint8)
    sigs = _sign_blocks(eng, sks, bits, msgs)
    rows = _rows(bits, 37)
    rows[:, 4] |= 0xE0
    assert eng.sync_aggregate_verify(np.zeros(3, dtype=np.uint32), rows, msgs, sigs).tolist() == [1, 1, 1]


# ------------------------------------------------------------------------------------------ two committees in one call
def test_two_committees_in_one_call(eng):
    size = 64
    sks0, pks0 = _committee(eng, size, 10000)
    sks1, pks1 = _committee(eng, size, 20000)
    eng.sync_committee_load(np.concatenate([pks0, pks1]), size)
    rng = np.random.default_rng(2)
    n = 40
    bits = [(rng.random(size) < rng.choice([0.2, 0.6, 0.97])).astype(np.uint8).tolist() for _ in range(n)]
    cidx = np.arange(n, dtype=np.uint32) % 2
    msgs = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    sigs = np.concatenate([_sign_blocks(eng, sks0 if c == 0 else sks1, [b], msgs[i:i + 1]) for i, (c, b) in enumerate(zip(cidx, bits))])
    rows = _rows(bits, size)
    assert eng.sync_aggregate_verify(cidx, rows, msgs, sigs).tolist() == [1] * n
    assert eng.sync_aggregate_verify(1 - cidx, rows, msgs, sigs).tolist() == [0] * n


# ------------------------------------------------------------------------------------------ mainnet size against FastAggregateVerify
MAINNET_SIZE, N_BLOCKS = 512, 8192


@pytest.fixture(scope="module")
def mainnet(eng):
    sks, pks = _committee(eng, MAINNET_SIZE, 30000)
    return sks, pks


@pytest.mark.parametrize("participation", [1.0, 0.95, 0.5])
def test_mainnet_size_matches_fast_aggregate_verify(eng, mainnet, participation):
    """one 512-key committee, 8 192 blocks, 1 % of them corrupted by a bit flipped after signing: the verdicts equal those of
    b2_fast_aggregate_verify given the committee's registry indices per block, and exactly the corrupted blocks are rejected"""
    sks, pks = mainnet
    eng.sync_committee_load(pks, MAINNET_SIZE)
    eng.registry_load(pks, np.full(MAINNET_SIZE, 32 * 10**9, dtype=np.uint64))
    rng = np.random.default_rng(int(participation * 100))
    bits = (rng.random((N_BLOCKS, MAINNET_SIZE)) < participation).astype(np.uint8)
    msgs = rng.integers(0, 256, size=(N_BLOCKS, 32), dtype=np.uint8)
    sk_arr = np.array(sks, dtype=object)
    sums = [int(sk_arr[b.astype(bool)].sum()) % R for b in bits]
    assert all(sums)
    sigs = eng.sign(sums, np.arange(N_BLOCKS, dtype=np.uint32), msgs)
    bad = rng.choice(N_BLOCKS, size=N_BLOCKS // 100, replace=False)
    for i in bad:
        bits[i, int(rng.integers(0, MAINNET_SIZE))] ^= 1
    rows = np.packbits(bits, axis=1, bitorder="little")
    want = np.ones(N_BLOCKS, dtype=np.uint8)
    want[bad] = 0
    members = np.tile(np.arange(MAINNET_SIZE, dtype=np.uint32), N_BLOCKS)
    off = (np.arange(N_BLOCKS + 1, dtype=np.uint64) * MAINNET_SIZE).astype(np.uint32)
    fav = eng.fast_aggregate_verify(members, off, rows, msgs, sigs)
    got = eng.sync_aggregate_verify(np.zeros(N_BLOCKS, dtype=np.uint32), rows, msgs, sigs)
    assert np.array_equal(fav, want)
    assert np.array_equal(got, want)
    assert _dev_verify(eng, np.zeros(N_BLOCKS, dtype=np.uint32), rows, msgs, sigs)[0] == want.tolist()
    if participation == 0.95:
        eng.set_verify_mode(True, bytes(range(32)))
        try:
            assert np.array_equal(eng.sync_aggregate_verify(np.zeros(N_BLOCKS, dtype=np.uint32), rows, msgs, sigs), want)
        finally:
            eng.set_verify_mode(False)


# ------------------------------------------------------------------------------------------ error contract and device guard
def test_rejected_calls_change_nothing():
    from pos_evolution_b200._lib import B2_EINVAL
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    try:
        sks, pks = _committee(e, 24, 40000)
        lib, h = e.lib, e.h
        bits = [[1] * 24, [1] * 10 + [0] * 14]
        msgs = np.zeros((2, 32), dtype=np.uint8)
        sigs = _sign_blocks(e, sks, bits, msgs)
        rows = _rows(bits, 24)
        ok = np.full(2, SENTINEL, dtype=np.uint8)
        pk = np.full((2, 48), SENTINEL, dtype=np.uint8)
        cidx = np.zeros(2, dtype=np.uint32)
        # no committee loaded yet
        assert lib.b2_sync_aggregate_verify(h, _p(cidx), _p(rows), _p(msgs), _p(sigs), 2, _p(ok), _p(pk)) == B2_EINVAL
        assert (ok == SENTINEL).all() and (pk == SENTINEL).all()
        e.sync_committee_load(pks, 24)
        before = e.sync_aggregate_verify(cidx, rows, msgs, sigs, want_pubkeys=True)
        assert before[0].tolist() == [1, 1]
        valid = np.full(1025, SENTINEL, dtype=np.uint8)
        big = np.tile(pks, (43, 1))[:1025]
        for rc in (lib.b2_sync_aggregate_verify(h, _p(np.array([0, 1], dtype=np.uint32)), _p(rows), _p(msgs), _p(sigs), 2, _p(ok), _p(pk)),
                   lib.b2_sync_aggregate_verify(h, _p(cidx), _p(rows), _p(msgs), None, 2, _p(ok), _p(pk)),
                   lib.b2_sync_aggregate_verify(h, _p(cidx), _p(rows), _p(msgs), _p(sigs), 0, _p(ok), _p(pk)),
                   lib.b2_sync_committee_load(h, _p(np.ascontiguousarray(big)), 1025, 1, _p(valid)),
                   lib.b2_sync_committee_load(h, None, 24, 2, _p(valid)),
                   lib.b2_sync_committee_load(h, _p(np.ascontiguousarray(pks)), 0, 1, _p(valid))):
            assert rc == B2_EINVAL
        assert (ok == SENTINEL).all() and (pk == SENTINEL).all() and (valid == SENTINEL).all()
        after = e.sync_aggregate_verify(cidx, rows, msgs, sigs, want_pubkeys=True)
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        # a successful load of other keys does replace the committee
        _, other = _committee(e, 24, 41000)
        e.sync_committee_load(other, 24)
        assert e.sync_aggregate_verify(cidx, rows, msgs, sigs).tolist() == [0, 0]
    finally:
        e.close()


def test_dev_guard(eng):
    """a committee index >= n_committees fails only its own block and sets B2_GUARD_BAD_INDEX; the flag is read and cleared once"""
    sks, pks = _committee(eng, 32, 50000)
    eng.sync_committee_load(pks, 32)
    bits = [[1] * 32, [0] * 32, [1] * 20 + [0] * 12, [1] * 5 + [0] * 27]
    msgs = np.zeros((4, 32), dtype=np.uint8)
    sigs = _sign_blocks(eng, sks, bits, msgs)
    sigs[1] = np.frombuffer(INF2, dtype=np.uint8)
    rows = _rows(bits, 32)
    assert eng.guard_flags() == 0
    assert _dev_verify(eng, [0, 0, 0, 0], rows, msgs, sigs)[0] == [1, 1, 1, 1]
    assert eng.guard_flags() == 0
    ok, pk = _dev_verify(eng, [0, 1, 0, 1 << 31], rows, msgs, sigs, want_pk=True)
    assert ok == [1, 0, 1, 0]                                                 # an empty block with a bad index is not "empty"
    assert bytes(pk[1]) == INF1
    assert eng.guard_flags() == 1
    assert eng.guard_flags() == 0


# ------------------------------------------------------------------------------------------ spec layer and facade against the oracle
def _state_to_product(PS, s):
    st = PS.BeaconState(
        slot=s.slot, fork=PS.Fork(s.fork.previous_version, s.fork.current_version, s.fork.epoch),
        genesis_validators_root=s.genesis_validators_root,
        validators=[PS.Validator(v.pubkey, v.effective_balance, v.slashed, v.activation_epoch, v.exit_epoch) for v in s.validators],
        balances=list(s.balances), randao_mixes=list(s.randao_mixes), block_roots=list(s.block_roots),
        previous_epoch_participation=list(s.previous_epoch_participation), current_epoch_participation=list(s.current_epoch_participation),
        previous_justified_checkpoint=PS.Checkpoint(s.previous_justified_checkpoint.epoch, s.previous_justified_checkpoint.root),
        current_justified_checkpoint=PS.Checkpoint(s.current_justified_checkpoint.epoch, s.current_justified_checkpoint.root),
        finalized_checkpoint=PS.Checkpoint(s.finalized_checkpoint.epoch, s.finalized_checkpoint.root))
    st.current_sync_committee = PS.SyncCommittee(list(s.current_sync_committee.pubkeys), s.current_sync_committee.aggregate_pubkey)
    st.next_sync_committee = PS.SyncCommittee(list(s.next_sync_committee.pubkeys), s.next_sync_committee.aggregate_pubkey)
    return st


def test_spec_matches_oracle(eng):
    from pos_evolution_b200 import spec as PS
    ospec, ostate, cur = SO.minimal_sync_state()
    pspec = PS.Spec(PS.MINIMAL, engine=eng)
    assert pspec.p.SYNC_COMMITTEE_SIZE == ospec.SYNC_COMMITTEE_SIZE == 32 and pspec.p.EPOCHS_PER_SYNC_COMMITTEE_PERIOD == 8
    assert PS.MAINNET.SYNC_COMMITTEE_SIZE == 512 and PS.MAINNET.EPOCHS_PER_SYNC_COMMITTEE_PERIOD == 256
    n = ospec.SYNC_COMMITTEE_SIZE
    patterns = {"all": [1] * n, "none": [0] * n, "half": [1, 0] * (n // 2), "dup_split": [1, 0] + [1] * (n - 2)}
    for name, bits in patterns.items():
        agg, _ = SO.honest_sync_aggregate(ospec, ostate, cur, bits)
        variants = [("honest", agg)]
        if name != "none":
            flipped = list(bits)
            flipped[7] ^= 1
            variants.append(("flipped", SO.SyncAggregate(flipped, agg.sync_committee_signature)))
        else:
            variants.append(("empty_other_sig", SO.SyncAggregate(bits, bytes(96))))
        for vname, a in variants:
            o = copy.deepcopy(ostate)
            try:
                ospec.process_sync_aggregate(o, a)
                want = ("ok", o.balances)
            except AssertionError:
                want = ("assert", None)
            p = _state_to_product(PS, ostate)
            try:
                pspec.process_sync_aggregate(p, PS.SyncAggregate(list(a.sync_committee_bits), a.sync_committee_signature))
                got = ("ok", p.balances)
            except AssertionError:
                got = ("assert", None)
            assert got == want, (name, vname)
            assert want[0] == ("ok" if vname == "honest" else "assert"), (name, vname)
    assert pspec.stats["sync_committee_uploads"] == 1                         # cached by content across the product states
    # the batched form: items of different slots / roots in one call
    p = _state_to_product(PS, ostate)
    items, want = [], []
    for slot in (3, 5, 8):
        root = ostate.block_roots[slot]
        msg = ospec.sync_signing_root(ostate, slot, root)
        bits = [1] * (n - slot) + [0] * slot
        sig = __import__("scenarios").sign_aggregate([v for v, b in zip(cur, bits) if b], msg)
        for r, s in ((root, sig), (bytes(32), sig)):
            items.append((slot, r, PS.SyncAggregate(bits, s)))
            want.append(int(SO.eth_fast_aggregate_verify([k for k, b in zip(ostate.current_sync_committee.pubkeys, bits) if b],
                                                         ospec.sync_signing_root(ostate, slot, r), s)))
    items.append((4, ostate.block_roots[4], PS.SyncAggregate([1] * (n - 1), sig)))           # wrong length
    want.append(0)
    assert pspec.verify_sync_aggregates(p, items).tolist() == want == [1, 0, 1, 0, 1, 0, 0]
    for e in (0, 7, 8, 15, 16):
        for v in (0, 3, 4, 11, 63):
            p.slot = ostate.slot
            if ospec.compute_sync_committee_period(e) <= 1:
                assert pspec.is_assigned_to_sync_committee(p, e, v) == ospec.is_assigned_to_sync_committee(ostate, e, v)
            else:
                with pytest.raises(AssertionError):
                    pspec.is_assigned_to_sync_committee(p, e, v)
        assert pspec.compute_sync_committee_period(e) == ospec.compute_sync_committee_period(e)


def test_bls_facade_matches_oracle(eng):
    from pos_evolution_b200 import bls
    bls.use_engine(eng)
    pks = [bc.registry()[0][bc.registry()[1]["pk%d" % i]] for i in (1, 2, 2)]
    sig = bc.sign(bc.sk(1) + 2 * bc.sk(2))
    neg = bc.registry()[0][bc.registry()[1]["neg1"]]
    cases = [(pks, sig), ([], INF2), ([], sig), ([], bytes(96)), ([pks[0], neg], INF2), (pks, INF2), (pks[:1], sig)]
    for keys, s in cases:
        assert bls.eth_fast_aggregate_verify(keys, bc.MSG, s) is SO.eth_fast_aggregate_verify(keys, bc.MSG, s), (len(keys), s[:2])
    assert bls.G2_POINT_AT_INFINITY == SO.G2_POINT_AT_INFINITY
    assert bls.eth_aggregate_pubkeys(pks) == SO.eth_aggregate_pubkeys(pks)
    assert bls.eth_aggregate_pubkeys([pks[0], neg]) == SO.eth_aggregate_pubkeys([pks[0], neg]) == INF1
    for bad in ([], [pks[0], INF1], [pks[0], bytes(48)]):
        with pytest.raises(AssertionError):
            bls.eth_aggregate_pubkeys(bad)
        with pytest.raises(AssertionError):
            SO.eth_aggregate_pubkeys(bad)
