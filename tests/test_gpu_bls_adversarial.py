"""The BLS kernels on adversarial inputs (tests/bls_cases.py), through every GPU path, byte for byte against the oracle:
bls.Aggregate (b2_aggregate), K2 in its TMA and LDG forms (b2_g1_aggregate), KeyValidate (b2_registry_load, b2_key_validate),
FastAggregateVerify on registry indices and on explicit keys in the team form, the thread form and RLC batches, and the epoch
path (b2_epoch_dev and the depth-3 pipeline in its thread, team, RLC and LDG-gather forms).  Run on an H100:
    python -m pytest tests/test_gpu_bls_adversarial.py -m gpu"""
import hashlib
import os

import numpy as np
import pytest

import bls_cases as bc
import scenarios
from oracle import bls_sig as B
from oracle import fast
from oracle.bls12_381 import R, E2, g2_compress, g2_decompress

pytestmark = pytest.mark.gpu

EFF = 32 * 10**9


def _engine(**env):
    """an Engine (environment knobs applied at b2_init only) with the case registry loaded; -> (engine, validity bytes)"""
    from pos_evolution_b200.engine import Engine
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        eng = Engine(0)
    finally:
        for k, v in saved.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    rows, _ = bc.registry()
    valid = eng.registry_load(np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(-1, 48), np.full(len(rows), EFF, dtype=np.uint64))
    return eng, valid


@pytest.fixture(scope="module")
def eng():
    e, _ = _engine()
    yield e
    e.close()


def _bits(rows, stride=None):
    n = max([len(r) for r in rows] + [1])
    stride = stride or (n + 7) // 8
    out = np.zeros((len(rows), stride), dtype=np.uint8)
    for a, r in enumerate(rows):
        for j, b in enumerate(r):
            if b:
                out[a, j >> 3] |= 1 << (j & 7)
    return out


def _u8(chunks, width):
    return np.frombuffer(b"".join(chunks), dtype=np.uint8).reshape(-1, width) if chunks else np.zeros((0, width), dtype=np.uint8)


def _signed_sum(names):
    """secret key of the sum of the registry keys `names` (pk<i>: +sk_i, neg<i>: -sk_i)"""
    k = 0
    for n in names:
        k += bc.sk(int(n[2:])) if n.startswith("pk") else -bc.sk(int(n[3:]))
    return k % R


# ------------------------------------------------------------------------------------------ bls.Aggregate
def test_aggregate_encodings_and_group_law(eng):
    encs = bc.g2_encodings()
    segs = [(name, [enc]) for name, enc in encs] + bc.g2_patterns()
    flat, off = [], [0]
    for _, s in segs:
        flat += s
        off.append(len(flat))
    out, status = eng.aggregate(_u8(flat, 96), off)
    for k, (name, s) in enumerate(segs):
        st, agg = bc.aggregate(s)
        assert (int(status[k]), bytes(out[k])) == (st, agg), name
    # a single canonical point round-trips exactly (sign bit included)
    for k, (name, enc) in enumerate(encs):
        if bc.decode_status(g2_decompress, enc) != 2:
            assert bytes(out[k]) == enc, name


# ------------------------------------------------------------------------------------------ K2, KeyValidate
def _g1_committees():
    rows, index = bc.registry()
    out = list(bc.g1_patterns())
    for name in index:                               # every row alone, and beside a valid key
        out.append(("row:" + name, [name], [1]))
        out.append(("pk19+" + name, ["pk19", name], [1, 1]))
    out.append(("torsion_shifted", ["pk1+t1", "pk2-t1"], [1, 1]))
    out.append(("nothing_selected", ["pk0", "enc:zero_bytes"], [0, 0]))
    out.append(("unselected_invalid", ["pk0", "enc:zero_bytes", "pk1"], [1, 0, 1]))
    return out


def _g1_batch(committees):
    _, index = bc.registry()
    members, off = [], [0]
    for _, names, _ in committees:
        members += [index[n] for n in names]
        off.append(len(members))
    return np.array(members, dtype=np.uint32), off, _bits([b for _, _, b in committees])


def test_g1_aggregate_tma_and_ldg(eng):
    rows, index = bc.registry()
    com = _g1_committees()
    members, off, bits = _g1_batch(com)
    want = [bc.g1_pattern_sum(rows, index, names, b) for _, names, b in com]
    eng_ldg, _ = _engine(B2_K2_TMA="0")
    try:
        for e in (eng, eng_ldg):
            out, status = e.g1_aggregate(members, off, bits)
            for a, (name, _, _) in enumerate(com):
                assert (int(status[a]), bytes(out[a])) == want[a], name
    finally:
        eng_ldg.close()


def test_registry_validity_and_key_validate(eng):
    rows, _ = bc.registry()
    e, valid = _engine()
    e.close()
    with bc.cached_key_validate():
        assert valid.tolist() == [int(B.KeyValidate(r)) for r in rows]
        keys = rows + [enc for _, enc in bc.g1_encodings() + bc.g1_boundary_encodings()]
        assert eng.key_validate(_u8(keys, 48)).tolist() == [int(B.KeyValidate(k)) for k in keys]


# ------------------------------------------------------------------------------------------ FastAggregateVerify
def _verify_cases():
    """[(name, registry names, bits, msg, sig)] for the registry path; the explicit-key path takes the selected keys' bytes"""
    _, index = bc.registry()
    out = []
    for name, enc in bc.g2_encodings():             # every signature encoding against the honest signer of sig "valid"
        out.append(("sig:" + name, ["pk0"], [1], bc.MSG, enc))
    for name, names, b in bc.g1_patterns():          # group-law committees, correctly signed by their selected keys
        sel = [n for n, x in zip(names, b) if x]
        out.append(("g1:" + name, names, b, bc.MSG, bc.sign(_signed_sum(sel))))
    for name in index:                               # every registry row beside a valid key, signed by that key alone
        if name.startswith("enc:"):
            out.append(("beside:" + name, ["pk19", name], [1, 1], bc.MSG, bc.sign(bc.sk(19))))
    out.append(("torsion_shifted", ["pk1+t1", "pk2-t1"], [1, 1], bc.MSG, bc.sign(bc.sk(1) + bc.sk(2))))
    out.append(("wrong_message", ["pk20"], [1], bc.MSG, bc.sign(bc.sk(20), bc.MSG2)))
    for c in bc.sharp_registry_cases():
        out.append(("sharp:" + c["name"], c["members"], c["bits"], c["msg"], c["sig"]))
    return out


@pytest.fixture(scope="module")
def verify_batch():
    """(registry batch, explicit-key batch, expected verdicts of each) -- the oracle runs once per module"""
    rows, index = bc.registry()
    cases = _verify_cases()
    members, off, bits = _g1_batch([(n, m, b) for n, m, b, _, _ in cases])
    msgs = _u8([c[3] for c in cases], 32)
    sigs = _u8([c[4] for c in cases], 96)
    want = []
    pk_lists = []
    for name, names, b, msg, sig in cases:
        sel = [rows[index[n]] for n, x in zip(names, b) if x]
        pk_lists.append(sel)
        want.append(int(bc.fav(sel, msg, sig)))
    names_x = [c[0] for c in cases]
    for c in bc.sharp_explicit_cases():
        pk_lists.append(c["pks"])
        names_x.append("sharp:" + c["name"])
    msgs_x = np.concatenate([msgs, _u8([c["msg"] for c in bc.sharp_explicit_cases()], 32)])
    sigs_x = np.concatenate([sigs, _u8([c["sig"] for c in bc.sharp_explicit_cases()], 96)])
    want_x = want + [int(bc.fav(c["pks"], c["msg"], c["sig"])) for c in bc.sharp_explicit_cases()]
    pk_off = np.cumsum([0] + [len(p) for p in pk_lists]).astype(np.uint32)
    pks = _u8([p for lst in pk_lists for p in lst], 48)
    assert 0 < sum(want) < len(want)
    return ([c[0] for c in cases], (members, off, bits, msgs, sigs), want), (names_x, (pks, pk_off, msgs_x, sigs_x), want_x)


def _check(got, names, want):
    bad = [(n, int(g), w) for n, g, w in zip(names, got, want) if int(g) != w]
    assert not bad, bad


@pytest.mark.parametrize("form", ["team", "thread", "rlc"])
def test_fast_aggregate_verify(eng, verify_batch, form):
    (names, reg, want), (names_x, expl, want_x) = verify_batch
    e = eng
    if form == "thread":
        e, _ = _engine(B2_PAIRING_FORM="thread")
    try:
        for seed in ((b"adv-seed-1", b"adv-seed-2") if form == "rlc" else (None,)):
            if seed:
                e.set_verify_mode(True, hashlib.sha256(seed).digest())
            try:
                _check(e.fast_aggregate_verify(*reg), names, want)
                _check(e.fast_aggregate_verify_pks(*expl), names_x, want_x)
            finally:
                if seed:
                    e.set_verify_mode(False)
    finally:
        if e is not eng:
            e.close()


def _rejected_outright():
    """aggregates every verification form rejects before the pairing: a bad key status, or an undecodable / non-G2 signature.
    The first three carry the signature infinity, so both Miller values are 1 and only the status test rejects them."""
    out = [(c["members"], c["bits"], c["sig"]) for c in bc.sharp_registry_cases() if c["sig"] == bc.INF2]
    out += [(["pk21"], [1], bytes(96)), (["pk21"], [1], dict(bc.g2_encodings())["not_in_g2"]),
            (["pk21", "enc:not_in_g1"], [1, 1], bc.sign(bc.sk(21)))]
    return out


def _honest(i):
    return (["pk%d" % (i % bc.N_HONEST)], [1], bc.sign(bc.sk(i % bc.N_HONEST)))


def _run_rlc_batch(eng, aggs, seed):
    rows, index = bc.registry()
    members, off, bits = _g1_batch([("", m, b) for m, b, _ in aggs])
    msgs = _u8([bc.MSG] * len(aggs), 32)
    want = [int(bc.fav([rows[index[n]] for n, x in zip(m, b) if x], bc.MSG, s)) for m, b, s in aggs]
    eng.set_verify_mode(True, hashlib.sha256(seed).digest())
    try:
        got = eng.fast_aggregate_verify(members, off, bits, msgs, _u8([s for _, _, s in aggs], 96)).tolist()
    finally:
        eng.set_verify_mode(False)
    return got, want


def test_rlc_group_placement(eng):
    """70 aggregates = groups of 32, 32 and 6; members rejected outright at both ends of every group, the rest honest: every group
    equation passes, so the rejected members are decided by the status tests of the RLC kernels alone"""
    rej = _rejected_outright()
    aggs = [_honest(i) for i in range(70)]
    for k, pos in enumerate((0, 31, 32, 63, 64, 69)):
        aggs[pos] = rej[k % len(rej)]
    got, want = _run_rlc_batch(eng, aggs, b"placement")
    assert want == [0 if a in (0, 31, 32, 63, 64, 69) else 1 for a in range(70)]
    assert got == want
    # group 0: every member rejected outright; group 1: one member fails only the equation (the fallback decides the group);
    # group 2: honest
    aggs = [rej[i % len(rej)] for i in range(32)] + [_honest(i) for i in range(32, 96)]
    aggs[45] = (["pk5"], [1], bc.sign(bc.sk(5), bc.MSG2))
    got, want = _run_rlc_batch(eng, aggs, b"groups")
    assert want == [0] * 32 + [1] * 13 + [0] + [1] * 50
    assert got == want


# ------------------------------------------------------------------------------------------ the epoch path
N_BLK = 40


def _epoch_committees():
    """[(name, registry names, bits, individual signatures)]: committee sizes 1, 32, 33, 513 and 0, the group-law and sharp cases.
    Each validator sits in one committee only, so the LMD table shows exactly which aggregates were accepted."""
    s = {i: bc.sign(bc.sk(i)) for i in range(bc.N_HONEST)}
    ns = {i: g2_compress(E2.neg(bc.sig_point(bc.sk(i)))) for i in (2, 4)}
    inf = bc.INF2
    t2 = bc.t2()
    out = [("size1", ["pk0"], [1], [s[0]]),
           ("size32_same", ["pk1"] * 32, [1] * 32, [s[1]] * 32),
           ("size33_alternating", ["pk2", "neg2"] * 16 + ["pk2"], [1] * 33, [s[2], ns[2]] * 16 + [s[2]]),
           ("size513_same", ["pk3"] * 513, [1] * 513, [s[3]] * 513),
           ("empty", [], [], []),
           ("halves_64", ["pk4"] * 32 + ["neg4"] * 32, [1] * 64, [s[4]] * 32 + [ns[4]] * 32),
           ("bits_subset", ["pk5", "pk6", "pk7"], [1, 0, 1], [s[5], inf, s[7]]),
           ("torsion_s_plus_t_and_s", ["pk20", "pk21"], [1, 1], [g2_compress(E2.add(bc.sig_point(bc.sk(20)), t2)), s[21]]),
           ("not_in_g2", ["pk22"], [1], [dict(bc.g2_encodings())["not_in_g2"]]),
           ("undecodable", ["pk23"], [1], [bytes(96)]),
           ("y_minus_s_plus_s", ["pk13", "pk14"], [1, 1], [p for n, p in bc.g2_patterns() if n.startswith("y_minus_s_plus_s:")][0])]
    for c in bc.sharp_aggregation_cases():
        out.append(("sharp:" + c["name"], c["members"], c["bits"], c["sigs"]))
    for c in bc.sharp_registry_cases():                # the first member signs, the others contribute the identity
        out.append(("sharp:" + c["name"], c["members"], c["bits"], [c["sig"]] + [inf] * (len(c["members"]) - 1)))
    return out


@pytest.fixture(scope="module")
def epoch_case():
    rows, index = bc.registry()
    com = _epoch_committees()
    members, off, bits = _g1_batch([(n, m, b) for n, m, b, _ in com])
    sigs = [x for _, _, _, ss in com for x in ss]
    want_agg, want_st, want_ok = [], [], []
    for name, names, b, ss in com:
        st, agg = bc.aggregate(ss)
        want_st.append(st)
        want_agg.append(agg)
        want_ok.append(int(st == 0 and bc.fav([rows[index[n]] for n, x in zip(names, b) if x], bc.MSG, agg)))
    assert 0 < sum(want_ok) < len(com)
    return [c[0] for c in com], members, np.array(off, dtype=np.uint32), bits, _u8(sigs, 96), want_agg, want_st, want_ok


@pytest.mark.parametrize("mode", ["sync", "sync_rlc", "pipelined_thread", "pipelined_team", "pipelined_rlc", "pipelined_ldg"])
def test_epoch_paths(epoch_case, mode):
    import torch
    from pos_evolution_b200.epoch import EpochProcessor
    names, members, off, bits, sigs, want_agg, want_st, want_ok = epoch_case
    n_agg, n_val = len(names), len(bc.registry()[0])
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 5)
    eng, _ = _engine(**({"B2_K2_TMA": "0"} if mode == "pipelined_ldg" else {}))
    dev = torch.device("cuda", 0)
    try:
        eng.tree_load(parent, slot, roots, leaf_viable)
        eng.latest_messages_reset()
        if mode.endswith("rlc"):
            eng.set_verify_mode(True, hashlib.sha256(b"epoch-" + mode.encode()).digest())
        ep = EpochProcessor(eng, n_agg, len(members), bits.shape[1], N_BLK, device=dev, depth=3,
                            tail_form="team" if mode == "pipelined_team" else "thread")
        ep.set_committees(members, off)
        m_epoch, m_block, m_has = np.zeros(n_val, np.uint64), np.zeros(n_val, np.uint32), np.zeros(n_val, np.uint8)
        zeros, eff = np.zeros(n_val, np.uint8), np.full(n_val, EFF, dtype=np.uint64)
        got, heads, keep = [], [], []

        def collect(t):
            ok, hd = t.wait()
            got.append((ok.cpu().numpy().tolist(), ep.d_agg_status[t.slot].cpu().numpy().tolist(), [bytes(r) for r in t.d_agg_sig.cpu().numpy()], hd))

        n_epochs = 1 if mode.startswith("sync") else 4
        for k in range(n_epochs):
            te = np.full(n_agg, 2 + k, dtype=np.int64)
            bi = ((np.arange(n_agg) * 7 + 3 * k) % N_BLK).astype(np.int32)
            for a in range(n_agg):
                if want_ok[a]:
                    fast.lmd_update(m_epoch, m_block, m_has, zeros, [int(members[off[a] + j]) for j in range(off[a + 1] - off[a]) if (bits[a, j >> 3] >> (j & 7)) & 1],
                                    2 + k, int(bi[a]))
            w = fast.ghost_weights(parent, m_block, m_has, eff, np.ones(n_val, np.uint8), zeros, -1, 0)
            heads.append(fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0))
            d = [torch.as_tensor(sigs.copy(), device=dev), torch.as_tensor(bits, device=dev),
                 torch.as_tensor(_u8([bc.MSG] * n_agg, 32).copy(), device=dev), torch.as_tensor(te, device=dev), torch.as_tensor(bi, device=dev)]
            keep.append(d)
            if mode.startswith("sync"):
                ok, hd = ep.process_epoch_dev(*d)
                torch.cuda.synchronize()
                got.append((ok.cpu().numpy().tolist(), ep.d_agg_status[0].cpu().numpy().tolist(), [bytes(r) for r in ep.d_agg_sig[0].cpu().numpy()],
                            int(hd.item())))
            else:
                t = ep.submit_dev(*d, last=(mode == "pipelined_team" and k == n_epochs - 1))
                if t is not None:
                    collect(t)
        for t in ep.drain():
            collect(t)
        assert len(got) == n_epochs
        for k, (ok, st, agg, hd) in enumerate(got):
            _check(ok, names, want_ok)
            assert st == want_st, k
            assert agg == want_agg, k
            assert hd == heads[k], k
        # rejected aggregates leave the LMD table untouched: it equals the sequential update by the accepted ones alone
        e, b, h = eng.latest_messages_read()
        assert np.array_equal(h, m_has) and np.array_equal(e[h == 1], m_epoch[h == 1]) and np.array_equal(b[h == 1], m_block[h == 1])
    finally:
        eng.close()
