"""bls.AggregateVerify and bls.AggregatePKs on the GPU (b2_aggregate_verify / _pks / _dev, b2_aggregate_pks; kernels in
csrc/aggverify.cuh): oracle parity on adversarial keys and signatures in all three forms, sets placed across every block boundary of
the per-item kernel, consistency with FastAggregateVerify, a 2^16-pair batch, the error contract, the device-side guards and the
facade.  Run on an H100:
    python -m pytest tests/test_gpu_aggregate_verify.py -m gpu"""
import ctypes
import hashlib

import numpy as np
import pytest

import bls_cases as bc
from oracle import bls_sig as B
from oracle.bls12_381 import E1, E2, g1_compress, g1_decompress, g2_compress

pytestmark = pytest.mark.gpu

EFF = 32 * 10**9
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    rows, _ = bc.registry()
    e.registry_load(_u8(rows, 48), np.full(len(rows), EFF, dtype=np.uint64))
    yield e
    e.close()


def _u8(chunks, width):
    return np.frombuffer(b"".join(chunks), dtype=np.uint8).reshape(-1, width) if chunks else np.zeros((0, width), dtype=np.uint8)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run_dev(eng, signer, msgs, off, sigs):
    import torch
    dev = torch.device("cuda", 0)
    d = [torch.as_tensor(np.array(x), device=dev) for x in (np.asarray(signer, dtype=np.uint32).astype(np.int32), msgs,
                                                                         np.asarray(off, dtype=np.uint32).astype(np.int32), sigs)]
    ok = torch.full((len(off) - 1,), 7, dtype=torch.uint8, device=dev)
    eng.aggregate_verify_dev(d[0], d[1], d[2], d[3], ok)
    torch.cuda.synchronize()
    return ok.cpu().numpy().tolist()


def _all_forms(eng, names, msgs, off, sigs):
    """verdicts of the registry, explicit-key and _dev forms for sets of registry names -> {form: [0/1]}"""
    rows, index = bc.registry()
    signer = np.array([index[n] for n in names], dtype=np.uint32)
    m, s = _u8(msgs, 32), _u8(sigs, 96)
    return {"registry": eng.aggregate_verify(signer, off, m, s).tolist(),
            "explicit": eng.aggregate_verify_pks(_u8([rows[i] for i in signer], 48), off, m, s).tolist(),
            "dev": _run_dev(eng, signer, m, off, s)}


def _flatten(sets):
    names, msgs, off = [], [], [0]
    for _, pairs, _ in sets:
        names += [n for n, _ in pairs]
        msgs += [m for _, m in pairs]
        off.append(len(names))
    return names, msgs, np.array(off, dtype=np.uint32), [s for _, _, s in sets]


# ------------------------------------------------------------------------------------------ oracle parity
def _parity_sets():
    """[(name, [(registry name, message)], signature)]"""
    M, M2 = bc.MSG, bc.MSG2
    s = lambda k, m=M: bc.sign(bc.sk(k), m)      # noqa: E731
    agg = lambda *sigs: B.Aggregate(list(sigs))    # noqa: E731
    out = [("empty_first", [], s(0)),
           ("duplicate_messages", [("pk0", M), ("pk1", M)], agg(s(0), s(1))),
           ("empty_between", [], bc.INF2),
           ("same_key_two_messages", [("pk2", M), ("pk2", M2)], agg(s(2), s(2, M2))),
           ("pk_and_neg_pk_infinity_sig", [("pk3", M), ("neg3", M)], bc.INF2),
           ("pk_and_neg_pk_two_messages", [("pk3", M), ("neg3", M2)], bc.INF2),
           ("wrong_message", [("pk4", M2)], s(4)),
           ("three_pairs", [("pk5", M), ("pk6", M2), ("pk7", M)], agg(s(5), s(6, M2), s(7)))]
    for name, _ in bc.g1_encodings():               # every key encoding beside an honest pair; the pairing alone accepts the first
        out.append(("key:%s:sig_without_it" % name, [("pk19", M), ("enc:" + name, M2)], s(19)))
        out.append(("key:%s:sig_with_pk0" % name, [("pk19", M), ("enc:" + name, M2)], agg(s(19), s(0, M2))))
    out.append(("torsion_shifted_keys", [("pk1+t1", M), ("pk2-t1", M)], bc.sign(bc.sk(1) + bc.sk(2))))
    for name, enc in bc.g2_encodings():             # every signature encoding under the key that signed "valid"
        out.append(("sig:" + name, [("pk0", M)], enc))
    out.append(("sig:s_plus_t2_two_pairs", [("pk8", M), ("pk9", M2)], g2_compress(E2.add(bc.sig_point(bc.sk(8)), bc.t2()))))
    out.append(("empty_last", [], bc.INF2))
    return out


@pytest.fixture(scope="module")
def parity_case():
    rows, index = bc.registry()
    sets = _parity_sets()
    with bc.cached_key_validate():
        want = [int(B.AggregateVerify([rows[index[n]] for n, _ in pairs], [m for _, m in pairs], sig)) for _, pairs, sig in sets]
    assert 0 < sum(want) < len(want)
    return sets, want


def test_oracle_parity_all_forms(eng, parity_case):
    sets, want = parity_case
    w = dict(zip([n for n, _, _ in sets], want))
    assert w["duplicate_messages"] == 1 and w["same_key_two_messages"] == 1 and w["key:valid:sig_with_pk0"] == 1
    got = _all_forms(eng, *_flatten(sets))
    for form, g in got.items():
        bad = [(n, v, x) for (n, _, _), v, x in zip(sets, g, want) if v != x]
        assert not bad, (form, bad)


# ------------------------------------------------------------------------------------------ block boundaries (GPU-built signatures)
SIZES = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 300)
N_KEYS = 512


@pytest.fixture(scope="module")
def keyed():
    """an engine with a registry of N_KEYS keys (secret keys 1000 + i) and a signer for batches of pairs"""
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    sks = [1000 + i for i in range(N_KEYS)]
    pks = e.sk_to_pk(sks)
    assert e.registry_load(pks, np.full(N_KEYS, EFF, dtype=np.uint64)).all()
    yield e, sks, pks
    e.close()


def _signed_batch(e, sks, sizes, seed, same_message=False):
    """(signer, msgs, off, aggregate signatures) of honest sets of the given sizes, signed on the GPU"""
    rng = np.random.default_rng(seed)
    off = np.cumsum([0] + list(sizes)).astype(np.uint32)
    n = int(off[-1])
    signer = rng.integers(0, N_KEYS, size=n).astype(np.uint32)
    msgs = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    if same_message:
        for s in range(len(sizes)):
            msgs[off[s]:off[s + 1]] = msgs[off[s]]
    sigs = e.sign([sks[i] for i in signer], np.arange(n, dtype=np.uint32), msgs) if n else np.zeros((0, 96), np.uint8)
    agg, st = e.aggregate(sigs, off)
    assert (st[np.diff(off) > 0] == 0).all()
    agg[np.diff(off) == 0] = np.frombuffer(bc.INF2, dtype=np.uint8)
    return signer, msgs, off, agg


def _verdicts(e, pks, signer, msgs, off, agg):
    got = {"registry": e.aggregate_verify(signer, off, msgs, agg).tolist(),
           "explicit": e.aggregate_verify_pks(pks[signer], off, msgs, agg).tolist(),
           "dev": _run_dev(e, signer, msgs, off, agg)}
    assert got["registry"] == got["explicit"] == got["dev"], got
    return got["registry"]


@pytest.mark.parametrize("shift", [0, 1, 17, 40, 63])
def test_block_boundaries(keyed, shift):
    """every set size around the 64-item block and the warp, behind `shift` one-pair sets so that runs start and end at many
    positions in a block; set s is honest (s % 5 == 0), has one bit of its first / middle / last message flipped (1, 2, 3), or
    carries its neighbour's signature (4)"""
    e, sks, pks = keyed
    rng = np.random.default_rng(shift)
    sizes = [1] * shift + list(rng.permutation(SIZES * 2))
    signer, msgs, off, agg = _signed_batch(e, sks, sizes, 100 + shift)
    n_sets = len(sizes)
    agg_honest = agg.copy()
    want = []
    for s in range(n_sets):
        mode, lo, hi = s % 5, int(off[s]), int(off[s + 1])
        if mode in (1, 2, 3):
            j = {1: lo, 2: (lo + hi - 1) // 2, 3: hi - 1}[mode]
            msgs[j, int(rng.integers(0, 32))] ^= np.uint8(1 << int(rng.integers(0, 8)))
        elif mode == 4:
            agg[s] = agg_honest[(s + 1) % n_sets]
        want.append(int(mode == 0))
    assert _verdicts(e, pks, signer, msgs, off, agg) == want


def test_consistency_with_fast_aggregate_verify_and_set_order(keyed):
    """sets whose messages are all equal: AggregateVerify == FastAggregateVerify on the same keys; permuting the sets permutes the
    verdicts"""
    e, sks, pks = keyed
    sizes = [1, 3, 33, 64, 65, 2, 129, 7]
    signer, msgs, off, agg = _signed_batch(e, sks, sizes, 7, same_message=True)
    agg[[1, 5]] = agg[[5, 1]]                    # two sets with a wrong signature
    msgs_per_set = msgs[off[:-1]]
    fav = e.fast_aggregate_verify_pks(pks[signer], off, msgs_per_set, agg).tolist()
    got = _verdicts(e, pks, signer, msgs, off, agg)
    assert got == fav == [1, 0, 1, 1, 1, 0, 1, 1]
    perm = np.random.default_rng(3).permutation(len(sizes))
    p_signer = np.concatenate([signer[off[s]:off[s + 1]] for s in perm])
    p_msgs = np.concatenate([msgs[off[s]:off[s + 1]] for s in perm])
    p_off = np.cumsum([0] + [sizes[s] for s in perm]).astype(np.uint32)
    assert _verdicts(e, pks, p_signer, p_msgs, p_off, agg[perm]) == [got[s] for s in perm]


def test_large_batch(keyed):
    """2^16 pairs in 2 048 sets of random sizes (some empty); every 7th non-empty set has one message bit flipped"""
    e, sks, pks = keyed
    rng = np.random.default_rng(16)
    cuts = np.sort(rng.integers(0, 1 << 16, size=2047))
    sizes = np.diff(np.concatenate([[0], cuts, [1 << 16]])).tolist()
    signer, msgs, off, agg = _signed_batch(e, sks, sizes, 16)
    want = []
    for s, n in enumerate(sizes):
        if n and s % 7 == 3:
            msgs[int(off[s]) + int(rng.integers(0, n)), 5] ^= np.uint8(0x10)
        want.append(int(n > 0 and s % 7 != 3))
    assert 0 in sizes
    got = e.aggregate_verify(signer, off, msgs, agg).tolist()
    assert got == want
    assert _run_dev(e, signer, msgs, off, agg) == want


# ------------------------------------------------------------------------------------------ error contract and device guards
def _state(e):
    return [*e.latest_messages_read()]


@pytest.mark.parametrize("case", ["signer_out_of_range", "decreasing_offsets", "null_signature", "pks_decreasing_offsets", "pks_null_keys",
                                  "aggregate_pks_decreasing_offsets"])
def test_rejected_call_changes_nothing(keyed, case):
    from pos_evolution_b200._lib import B2_EINVAL
    e, sks, pks = keyed
    lib, h = e.lib, e.h
    signer, msgs, off, agg = _signed_batch(e, sks, [2, 3, 1], 5)
    before_ok = e.aggregate_verify(signer, off, msgs, agg).tolist()
    before = _state(e)
    out = np.full(3, SENTINEL, dtype=np.uint8)
    out48 = np.full((3, 48), SENTINEL, dtype=np.uint8)
    k = np.array(pks[signer])
    if case == "signer_out_of_range":
        bad = signer.copy()
        bad[4] = N_KEYS
        rc = lib.b2_aggregate_verify(h, _p(bad), _p(msgs), _p(off), _p(agg), 3, _p(out))
    elif case == "decreasing_offsets":
        rc = lib.b2_aggregate_verify(h, _p(signer), _p(msgs), _p(np.array([0, 4, 2, 6], dtype=np.uint32)), _p(agg), 3, _p(out))
    elif case == "null_signature":
        rc = lib.b2_aggregate_verify(h, _p(signer), _p(msgs), _p(off), None, 3, _p(out))
    elif case == "pks_decreasing_offsets":
        rc = lib.b2_aggregate_verify_pks(h, _p(k), _p(msgs), _p(np.array([0, 4, 2, 6], dtype=np.uint32)), _p(agg), 3, _p(out))
    elif case == "pks_null_keys":
        rc = lib.b2_aggregate_verify_pks(h, None, _p(msgs), _p(off), _p(agg), 3, _p(out))
    else:
        rc = lib.b2_aggregate_pks(h, _p(k), _p(np.array([0, 4, 2, 6], dtype=np.uint32)), 3, _p(out48), _p(out))
    assert rc == B2_EINVAL
    assert (out == SENTINEL).all() and (out48 == SENTINEL).all()
    for a, b in zip(before, _state(e)):
        assert np.array_equal(a, b)
    assert e.aggregate_verify(signer, off, msgs, agg).tolist() == before_ok == [1, 1, 1]


def test_dev_guards(keyed):
    """a signer index >= n_validators fails only its own set (B2_GUARD_BAD_INDEX); malformed offsets fail every set of the call
    (B2_GUARD_BAD_ROW); b2_guard_flags returns and clears the word"""
    from pos_evolution_b200._lib import B2_OK
    e, sks, pks = keyed
    signer, msgs, off, agg = _signed_batch(e, sks, [3, 2, 4, 1], 9)
    assert e.guard_flags() == 0
    assert _run_dev(e, signer, msgs, off, agg) == [1, 1, 1, 1]
    assert e.guard_flags() == 0
    bad = signer.copy()
    bad[3] = N_KEYS + 5                               # set 1
    assert _run_dev(e, bad, msgs, off, agg) == [1, 0, 1, 1]
    assert e.guard_flags() == 1
    assert e.guard_flags() == 0
    for o in ([1, 3, 5, 9, 10], [0, 3, 2, 9, 10], [0, 3, 5, 9, 11]):     # off[0] != 0, a decreasing pair, past the pairs
        assert _run_dev(e, signer, msgs, np.array(o, dtype=np.uint32), agg) == [0, 0, 0, 0]
        assert e.guard_flags() == 2
    assert _run_dev(e, signer[:9], msgs[:9], np.array([0, 3, 5, 9, 9], dtype=np.uint32), agg) == [1, 1, 1, 0]      # fewer pairs, in bounds
    bad_both = signer.copy()
    bad_both[0] = 1 << 31
    assert _run_dev(e, bad_both, msgs, off, agg) == [0, 1, 1, 1]
    assert _run_dev(e, signer, msgs, np.array([0, 3, 2, 9, 10], dtype=np.uint32), agg) == [0, 0, 0, 0]
    f = ctypes.c_uint32(0)
    assert e.lib.b2_guard_flags(e.h, ctypes.byref(f)) == B2_OK and f.value == 3
    assert e.guard_flags() == 0


# ------------------------------------------------------------------------------------------ AggregatePKs
def test_aggregate_pks_matches_oracle(eng):
    rows, index = bc.registry()
    pk = lambda n: rows[index[n]]                   # noqa: E731
    segs = [[pk("pk0")], [pk("pk0"), pk("pk1"), pk("pk2")], [pk("pk3"), pk("neg3")], [pk("pk4")] * 33, [pk("pk5"), pk("pk5"), pk("neg5")]]
    bad = [[], [pk("pk0"), pk("enc:not_in_g1")], [pk("enc:infinity")], [pk("enc:zero_bytes"), pk("pk1")]]
    off = np.cumsum([0] + [len(s) for s in segs + bad]).astype(np.uint32)
    out, status = eng.aggregate_pks(_u8([k for s in segs + bad for k in s], 48), off)
    with bc.cached_key_validate():
        for a, s in enumerate(segs):
            assert bytes(out[a]) == B.AggregatePKs(s), a
            assert (int(status[a]) & 3) == 0, a
        for a, s in enumerate(bad, start=len(segs)):
            with pytest.raises(ValueError):
                B.AggregatePKs(s)
            assert int(status[a]) & 3, a
    assert bytes(out[2]) == bc.INF1 and int(status[2]) == 4


# ------------------------------------------------------------------------------------------ the bls facade
def test_facade():
    from pos_evolution_b200 import bls
    M, M2 = bc.MSG, bc.MSG2
    pks = [B.SkToPk(bc.sk(k)) for k in (10, 11)]
    sig = B.Aggregate([bc.sign(bc.sk(10), M), bc.sign(bc.sk(11), M2)])
    assert bls.AggregateVerify(pks, [M, M2], sig) is True
    assert bls.AggregateVerify(pks, [M2, M], sig) is False
    assert bls.AggregateVerify(pks, [M, M], bc.sign(bc.sk(10) + bc.sk(11))) is True         # messages need not be distinct
    for args in (([], [], sig), (pks, [M], sig), (pks[:1], [M, M2], sig), ([pks[0][:47], pks[1]], [M, M2], sig), (pks, [M, M2], sig[:95]),
                 ([bc.INF1, pks[1]], [M, M2], sig), (pks, [M, M2], bytes(96)), (None, [M], sig), (pks, None, sig), (pks, [M, M2], None)):
        assert bls.AggregateVerify(*args) is False, args
    with pytest.raises(ValueError):
        bls.AggregateVerify(pks, [M, M2[:31]], sig)
    with pytest.raises(ValueError):
        bls.AggregateVerify(pks, [M, M2 + b"\x00"], sig)
    neg = g1_compress(E1.neg(g1_decompress(pks[0])))
    assert bls.AggregatePKs(pks) == B.AggregatePKs(pks)
    assert bls.AggregatePKs([pks[0], neg]) == B.AggregatePKs([pks[0], neg]) == bc.INF1
    assert bls._AggregatePKs(pks) == bls.AggregatePKs(pks)
    for bad in ([], [pks[0], bc.INF1], [pks[0], bytes(48)], [pks[0][:47]], [dict(bc.g1_encodings())["not_in_g1"]]):
        with pytest.raises(ValueError):
            bls.AggregatePKs(bad)
