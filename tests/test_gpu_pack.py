"""GPU block packing (b2_pack_attestations / _dev, Spec.get_attestations_for_block) against tests/pack_oracle.py, byte for byte on every
output field: committee, data id, union row, numerator, constituents, signature, candidate status."""
import copy
import ctypes

import numpy as np
import pytest

import pack_oracle as PO
import scenarios
from oracle import bls_sig as OB
from oracle import spec as OS
from oracle.bls12_381 import G1, g1_compress

pytestmark = pytest.mark.gpu

BAD_SIG = bytes([0x00]) + bytes(95)                       # compression flag missing: never decodes


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _load(eng, pool):
    n = len(pool["eff"])
    eng.registry_load(np.tile(np.frombuffer(g1_compress(G1), dtype=np.uint8), (n, 1)), pool["eff"])
    eng.participation_load(0, pool["part"][0])
    eng.participation_load(1, pool["part"][1])


def _sigs(eng, pool):
    """a real signature per decodable candidate (sk = c + 1 on the message of its data id), BAD_SIG elsewhere"""
    n = len(pool["comm"])
    if n == 0:
        return np.zeros((0, 96), dtype=np.uint8)
    msgs = np.frombuffer(b"".join(bytes([d & 255, d >> 8]) + bytes(30) for d in range(n)), dtype=np.uint8).reshape(n, 32)
    sigs = eng.sign(list(range(1, n + 1)), np.asarray(pool["data"], dtype=np.uint32), msgs)
    for c in range(n):
        if not pool["ok"][c]:
            sigs[c] = np.frombuffer(BAD_SIG, dtype=np.uint8)
    return sigs


def _run(eng, pool, sigs):
    return eng.pack_attestations(pool["members"], pool["off"], pool["table"], pool["comm"], pool["data"], pool["mask"], pool["bits"], sigs,
                                 pool["max_out"], pool["inc"], pool["per_inc"])


def _check(eng, pool, sigs, res, picks, oracle_sigs=True):
    stride = pool["bits"].shape[1]
    assert len(res.committee) == len(picks)
    assert res.cand_status.tolist() == [0 if ok else 1 for ok in pool["ok"]]
    off = [0]
    for o, (k, d, row, g, src) in enumerate(picks):
        assert int(res.committee[o]) == k and int(res.data[o]) == d and int(res.numerator[o]) == g
        assert res.bits[o].tobytes() == PO.row_bytes(row, stride)
        off.append(off[-1] + len(src))
        assert tuple(int(x) for x in res.src[off[o]:off[o + 1]]) == src
    assert res.src_off.tolist() == off
    if not picks:
        return
    multi = [o for o, p in enumerate(picks) if len(p[4]) > 1]
    for o, p in enumerate(picks):
        if len(p[4]) == 1:
            assert res.signature[o].tobytes() == sigs[p[4][0]].tobytes()
    if multi:
        flat = np.concatenate([sigs[list(picks[o][4])] for o in multi])
        seg = np.cumsum([0] + [len(picks[o][4]) for o in multi]).astype(np.uint32)
        agg, st = eng.aggregate(flat, seg)
        assert st.tolist() == [0] * len(multi)
        for i, o in enumerate(multi):
            assert res.signature[o].tobytes() == agg[i].tobytes()
            if oracle_sigs and i < 3:
                assert res.signature[o].tobytes() == OB.Aggregate([sigs[c].tobytes() for c in picks[o][4]])


CASES = {
    "small": dict(seed=1),
    "max_out_below": dict(seed=2, max_out=2),
    "max_out_above": dict(seed=3, max_out=500),
    "tie_heavy": dict(seed=4, tie_heavy=True, n_val=128, comms=(4, 4), n_cand=120, max_out=40),
    "tie_heavy_2": dict(seed=5, tie_heavy=True, n_val=64, comms=(2, 2), n_cand=80, max_out=7),
    "one_table": dict(seed=6, comms=(8, 0)),
    "previous_only": dict(seed=7, comms=(0, 6)),
    "undecodable": dict(seed=8, bad_frac=0.3, n_cand=100, max_out=30),
    "singles": dict(seed=9, singles=0.9, n_cand=150, max_out=20),
    "wide_2048": dict(seed=10, n_val=4096, comms=(2, 2), n_cand=60, max_out=12),
    "stride_pad": dict(seed=11, stride=256, max_out=10),
    "spill": dict(seed=12, n_val=2048, comms=(1, 0), n_cand=700, max_out=64, singles=0.5),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_pack_matches_oracle(eng, case):
    kw = dict(CASES[case])
    pool = PO.random_pool(kw.pop("seed"), **kw)
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    part0, part1 = eng.participation_read(0), eng.participation_read(1)
    res = _run(eng, pool, sigs)
    picks = PO.pack_literal(pool) if len(pool["comm"]) <= 200 else PO.pack_per_committee(pool)
    assert picks == PO.pack_per_committee(pool)
    _check(eng, pool, sigs, res, picks)
    # the device tables are unchanged, and process_attestation's bookkeeping over the picks credits exactly the numerators
    assert np.array_equal(eng.participation_read(0), part0) and np.array_equal(eng.participation_read(1), part1)
    for t in (0, 1):
        sel = [o for o in range(len(picks)) if int(pool["table"][picks[o][0]]) == t]
        if not sel:
            continue
        mem, off, rows, masks = [], [0], [], []
        for o in sel:
            k = picks[o][0]
            mem += pool["members"][pool["off"][k]:pool["off"][k + 1]].tolist()
            off.append(len(mem))
            rows.append(res.bits[o])
            masks.append(pool["mask"][res.src[res.src_off[o]]])
        num = eng.participation_update(t, mem, off, np.stack(rows), masks, None, pool["inc"], pool["per_inc"])
        assert [int(x) for x in num] == [int(res.numerator[o]) for o in sel]


def test_empty_pool_and_zero_gains(eng):
    pool = PO.random_pool(20, n_cand=0)
    _load(eng, pool)
    res = _run(eng, pool, np.zeros((0, 96), dtype=np.uint8))
    assert len(res.committee) == 0 and res.src_off.tolist() == [0] and len(res.cand_status) == 0
    pool = PO.random_pool(21, n_cand=50)
    pool["part"] = [np.full(len(pool["eff"]), 7, dtype=np.uint8)] * 2                 # every flag set: nothing earns
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    res = _run(eng, pool, sigs)
    assert len(res.committee) == 0 and PO.pack_literal(pool) == []
    assert res.cand_status.tolist() == [0] * 50


def test_single_bits_fold_to_one(eng):
    pool = PO.random_pool(22, n_val=64, comms=(1, 0), n_cand=0, max_out=4)
    size = int(pool["off"][1])
    bits = np.zeros((size, (size + 7) // 8), dtype=np.uint8)
    for j in range(size):
        bits[j, j >> 3] = 1 << (j & 7)
    pool.update(comm=np.zeros(size, dtype=np.uint32), data=np.zeros(size, dtype=np.uint32), mask=np.full(size, 7, dtype=np.uint8), bits=bits,
                ok=[True] * size)
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    res = _run(eng, pool, sigs)
    picks = PO.pack_literal(pool)
    assert len(picks) == 1 and picks[0][4] == tuple(range(size))
    _check(eng, pool, sigs, res, picks)


def test_mainnet_size_pool(eng):
    """2^20 validators, 2 048 committees of 512 per table (both tables), about six candidates per committee, against the per-committee
    oracle (vectorised per committee)"""
    rng = np.random.default_rng(30)
    n_val, per_table, size = 1 << 20, 2048, 512
    eff = rng.choice([16, 24, 31, 32, 32, 32], size=n_val).astype(np.uint64) * np.uint64(10**9)
    part = [(rng.integers(0, 8, size=n_val) * (rng.random(n_val) < 0.5)).astype(np.uint8) for _ in range(2)]
    members = np.concatenate([rng.permutation(n_val) for _ in range(2)]).astype(np.uint32)
    off = np.arange(0, 2 * n_val + 1, size, dtype=np.uint32)
    K = 2 * per_table
    comm = np.repeat(np.arange(K, dtype=np.uint32), 6)
    C = len(comm)
    data = (comm * 2 + (rng.random(C) < 0.2)).astype(np.uint32)
    data = np.unique(data, return_inverse=True)[1].astype(np.uint32)
    vote_mask = rng.integers(1, 8, size=int(data.max()) + 1).astype(np.uint8)
    rows = rng.random((C, size)) < rng.choice([0.1, 0.6, 0.9], size=(C, 1))
    bits = np.packbits(rows, axis=1, bitorder="little")
    pool = {"members": members, "off": off, "table": np.repeat(np.arange(2, dtype=np.uint8), per_table), "comm": comm, "data": data,
            "mask": vote_mask[data], "bits": bits, "ok": [True] * C, "eff": eff, "part": part, "inc": 10**9, "per_inc": 977, "max_out": 128}
    eng.registry_load(np.tile(np.frombuffer(g1_compress(G1), dtype=np.uint8), (n_val, 1)), eff)
    eng.participation_load(0, part[0])
    eng.participation_load(1, part[1])
    sigs = eng.sign(list(range(1, C + 1)), np.zeros(C, dtype=np.uint32), np.zeros((1, 32), dtype=np.uint8))
    res = _run(eng, pool, sigs)
    picks = PO.pack_per_committee(pool)
    assert len(picks) == 128
    _check(eng, pool, sigs, res, picks, oracle_sigs=False)


def test_dev_equals_host(eng):
    import torch
    pool = PO.random_pool(40, n_cand=150, max_out=25, bad_frac=0.1, comms=(5, 3))
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    res = _run(eng, pool, sigs)
    d = _dev_tensor
    C, M, stride = len(pool["comm"]), pool["max_out"], pool["bits"].shape[1]
    outs = [torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(M, dtype=torch.int32, device="cuda"),
            torch.zeros(M, dtype=torch.int32, device="cuda"), torch.zeros((M, stride), dtype=torch.uint8, device="cuda"),
            torch.zeros((M, 96), dtype=torch.uint8, device="cuda"), torch.zeros(M, dtype=torch.int64, device="cuda"),
            torch.zeros(M + 1, dtype=torch.int32, device="cuda"), torch.zeros(C, dtype=torch.int32, device="cuda"),
            torch.zeros(C, dtype=torch.uint8, device="cuda")]
    eng.pack_attestations_dev(d(pool["members"], np.uint32), d(pool["off"], np.uint32), d(pool["table"], np.uint8), d(pool["comm"], np.uint32),
                              d(pool["data"], np.uint32), d(pool["mask"], np.uint8), d(pool["bits"], np.uint8), d(sigs, np.uint8), M, pool["inc"],
                              pool["per_inc"], *outs)
    torch.cuda.synchronize()
    h = [t.cpu().numpy() for t in outs]
    n = int(h[0][0])
    assert n == len(res.committee) and eng.guard_flags() == 0
    assert np.array_equal(h[1][:n].view(np.uint32), res.committee) and np.array_equal(h[2][:n].view(np.uint32), res.data)
    assert np.array_equal(h[3][:n], res.bits) and np.array_equal(h[4][:n], res.signature)
    assert np.array_equal(h[5][:n].view(np.uint64), res.numerator) and np.array_equal(h[6][:n + 1].view(np.uint32), res.src_off)
    assert np.array_equal(h[7][:int(res.src_off[-1])].view(np.uint32), res.src) and np.array_equal(h[8], res.cand_status)
    assert not h[3][n:].any() and not h[4][n:].any() and not h[5][n:].any() and (h[6][n:] == res.src_off[-1]).all()


def _dev_tensor(a, dt):
    import torch
    a = np.ascontiguousarray(a, dtype=dt)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()


def _sentinel(shape, dt):
    return np.full(int(np.prod(shape)) * np.dtype(dt).itemsize, 0xAB, dtype=np.uint8).view(dt).reshape(shape)


def _raw_call(eng, pool, sigs, **over):
    """b2_pack_attestations with sentinel-filled outputs -> (rc, outputs)"""
    a = {k: np.ascontiguousarray(v) for k, v in dict(members=pool["members"], off=pool["off"], table=pool["table"], comm=pool["comm"],
                                                      data=pool["data"], mask=pool["mask"], bits=pool["bits"], sigs=sigs).items()}
    a.update({k: np.ascontiguousarray(v) for k, v in over.items() if k in a})
    M, C, stride = over.get("max_out", pool["max_out"]), len(pool["comm"]), pool["bits"].shape[1]
    m = max(M, 1)
    outs = [_sentinel((1,), np.uint32), _sentinel((m,), np.uint32), _sentinel((m,), np.uint32), _sentinel((m, stride), np.uint8),
            _sentinel((m, 96), np.uint8), _sentinel((m,), np.uint64), _sentinel((m + 1,), np.uint32), _sentinel((C,), np.uint32),
            _sentinel((C,), np.uint8)]
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)     # noqa: E731
    rc = eng.lib.b2_pack_attestations(eng.h, p(a["members"]), p(a["off"]), p(a["table"]), len(a["off"]) - 1, p(a["comm"]), p(a["data"]), p(a["mask"]),
                                      p(a["bits"]), over.get("stride", stride), p(a["sigs"]), C, M, pool["inc"], pool["per_inc"], *[p(o) for o in outs])
    return rc, outs


def test_error_contract(eng):
    from pos_evolution_b200._lib import B2_EINVAL
    pool = PO.random_pool(50, n_val=128, comms=(4, 4), n_cand=40, max_out=8)
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    overlap = pool["members"].copy()
    overlap[1] = overlap[40]                                                   # committees 0 and 1 of table 0 share a member
    big = pool["comm"].copy()
    big[3] = len(pool["table"])
    data_far = pool["data"].copy()
    data_far[0] = 10**6
    two_comm = pool["data"].copy()
    j = int(np.nonzero(pool["comm"] != pool["comm"][0])[0][0])
    two_comm[j] = pool["data"][0]                                               # one data id, two committees
    two_mask = pool["mask"].copy()
    same = [c for c in range(1, 40) if pool["data"][c] == pool["data"][0]]
    bad_members = pool["members"].copy()
    bad_members[5] = 128
    table2 = pool["table"].copy()
    table2[0] = 2
    cases = [dict(members=overlap), dict(comm=big), dict(data=data_far), dict(data=two_comm), dict(max_out=0), dict(members=bad_members),
             dict(table=table2), dict(stride=1)]
    if same:
        two_mask[same[0]] = two_mask[0] ^ 1
        cases.append(dict(mask=two_mask))
    for over in cases:
        rc, outs = _raw_call(eng, pool, sigs, **over)
        assert rc == B2_EINVAL, over.keys()
        assert all((o.view(np.uint8) == 0xAB).all() for o in outs), over.keys()
    rc, outs = _raw_call(eng, pool, sigs)
    assert rc == 0 and int(outs[0][0]) == len(PO.pack_literal(pool))
    from pos_evolution_b200.engine import Engine
    e2 = Engine(0)                                                             # no registry
    rc, outs = _raw_call(e2, pool, sigs)
    assert rc == B2_EINVAL and all((o.view(np.uint8) == 0xAB).all() for o in outs)
    e2.close()


def test_dev_guards(eng):
    import torch
    pool = PO.random_pool(60, n_val=128, comms=(4, 4), n_cand=40, max_out=8)
    _load(eng, pool)
    sigs = _sigs(eng, pool)
    d = _dev_tensor

    def run(p):
        C, M, stride = len(p["comm"]), p["max_out"], p["bits"].shape[1]
        outs = [torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(M, dtype=torch.int32, device="cuda"),
                torch.zeros(M, dtype=torch.int32, device="cuda"), torch.zeros((M, stride), dtype=torch.uint8, device="cuda"),
                torch.zeros((M, 96), dtype=torch.uint8, device="cuda"), torch.zeros(M, dtype=torch.int64, device="cuda"),
                torch.zeros(M + 1, dtype=torch.int32, device="cuda"), torch.zeros(C, dtype=torch.int32, device="cuda"),
                torch.zeros(C, dtype=torch.uint8, device="cuda")]
        eng.pack_attestations_dev(d(p["members"], np.uint32), d(p["off"], np.uint32), d(p["table"], np.uint8), d(p["comm"], np.uint32),
                                  d(p["data"], np.uint32), d(p["mask"], np.uint8), d(p["bits"], np.uint8), d(sigs, np.uint8), M, p["inc"], p["per_inc"],
                                  *outs)
        flags = eng.guard_flags()
        return int(outs[0].item()), outs[8].cpu().numpy(), flags

    # a bad committee index excludes that candidate only
    p = dict(pool)
    p["comm"] = pool["comm"].copy()
    p["comm"][3] = 10**6
    ref = dict(pool)
    ref["ok"] = [ok and c != 3 for c, ok in enumerate(pool["ok"])]
    n, status, flags = run(p)
    assert flags == 1 and status[3] == 2 and n == len(PO.pack_literal(ref))
    # overlap inside a table, and an inconsistent data id: the call selects nothing
    p = dict(pool)
    p["members"] = pool["members"].copy()
    p["members"][1] = p["members"][40]
    n, _, flags = run(p)
    assert n == 0 and flags == 8
    p = dict(pool)
    p["data"] = pool["data"].copy()
    j = int(np.nonzero(pool["comm"] != pool["comm"][0])[0][0])
    p["data"][j] = pool["data"][0]
    n, _, flags = run(p)
    assert n == 0 and flags == 8
    n, _, flags = run(pool)
    assert n == len(PO.pack_literal(pool)) and flags == 0


def test_spec_get_attestations_for_block(eng):
    """real signatures: get_attestations_for_block -> process_attestations on a copy of the state succeeds, the proposer's balance grows
    by sum(numerator // denominator), and the list is the oracle packing"""
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from test_gpu_spec import _state_to_product, _to_product
    pks = scenarios.pubkeys(64)
    ospec, ostate = scenarios.minimal_state(64, slot=12, pks=pks)
    rng = np.random.default_rng(70)
    ostate.current_epoch_participation = [int(x) for x in (rng.integers(0, 8, size=64) * (rng.random(64) < 0.3))]
    state = _state_to_product(PS, ostate)
    spec = PS.Spec(PS.MINIMAL, engine=Engine(0))
    signer = spec.engine
    cur = spec.get_current_epoch(state)
    pool = []
    for slot in range(4, 12):
        for index in range(spec.get_committee_count_per_slot(state, spec.compute_epoch_at_slot(slot))):
            committee = spec.get_beacon_committee(state, slot, index)
            for head in (None, b"\x22" * 32):
                for _ in range(2):
                    bits = [bool(b) for b in (rng.random(len(committee)) < 0.5)]
                    if not any(bits):
                        bits[0] = True
                    a = _to_product(PS, _unsigned(ospec, ostate, slot, index, bits, head))
                    signers = [v for v, b in zip(committee, bits) if b]
                    msg = spec.compute_signing_root(a.data, spec.get_domain(state, PS.DOMAIN_BEACON_ATTESTER, a.data.target.epoch))
                    s = signer.sign([scenarios.secret_key(v) for v in signers], [0] * len(signers), np.frombuffer(msg, dtype=np.uint8).reshape(1, 32))
                    agg, st = signer.aggregate(s, [0, len(signers)])
                    a.signature = agg[0].tobytes()
                    pool.append(a)
    pool.append(PS.Attestation([True] * 4, pool[0].data, bytes(96)))           # undecodable: never chosen
    out = spec.get_attestations_for_block(state, pool, 5)
    assert 0 < len(out) <= 5
    # the oracle packing of the same pool
    per_inc = spec.get_base_reward_per_increment(state)
    comms, dids, datas, members, off, table, oc, od, om, rows, ok = {}, {}, [], [], [0], [], [], [], [], [], []
    for a in pool:
        committee, flags = spec._check_attestation(state, a)
        key = (a.data.slot, a.data.index)
        if key not in comms:
            comms[key] = len(table)
            members += committee
            off.append(len(members))
            table.append(0 if a.data.target.epoch == cur else 1)
        r = PS.hash_tree_root_attestation_data(a.data)
        if r not in dids:
            dids[r] = len(datas)
            datas.append(a.data)
        oc.append(comms[key])
        od.append(dids[r])
        om.append(sum(1 << f for f in flags))
        rows.append(PS.pack_bits([a.aggregation_bits], stride=1)[0])
        ok.append(a.signature != bytes(96))
    opool = {"members": members, "off": off, "table": table, "comm": oc, "data": od, "mask": om, "bits": np.stack(rows), "ok": ok,
             "eff": [v.effective_balance for v in state.validators], "part": (state.current_epoch_participation, state.previous_epoch_participation),
             "inc": PS.MINIMAL.EFFECTIVE_BALANCE_INCREMENT, "per_inc": per_inc, "max_out": 5}
    picks = PO.pack_literal(opool)
    assert [(comms[(a.data.slot, a.data.index)], dids[PS.hash_tree_root_attestation_data(a.data)]) for a in out] == [(p[0], p[1]) for p in picks]
    assert [PS.pack_bits([a.aggregation_bits], stride=1)[0].tobytes() for a in out] == [PO.row_bytes(p[2], 1) for p in picks]
    for a, p in zip(out, picks):
        if len(p[4]) > 1:
            assert a.signature == OB.Aggregate([pool[c].signature for c in p[4]])
    st2 = copy.deepcopy(state)
    proposer = spec.get_beacon_proposer_index(st2)
    bal0 = st2.balances[proposer]
    spec.process_attestations(st2, out)
    denominator = (PS.WEIGHT_DENOMINATOR - PS.PROPOSER_WEIGHT) * PS.WEIGHT_DENOMINATOR // PS.PROPOSER_WEIGHT
    assert st2.balances[proposer] - bal0 == sum(p[3] // denominator for p in picks)
    spec.engine.close()


def _unsigned(ospec, ostate, slot, index, bits, head_root):
    epoch = ospec.compute_epoch_at_slot(slot)
    cur = ospec.get_current_epoch(ostate)
    just = ostate.current_justified_checkpoint if epoch == cur else ostate.previous_justified_checkpoint
    target = OS.Checkpoint(epoch, ospec.get_block_root(ostate, epoch))
    head = head_root if head_root is not None else ospec.get_block_root_at_slot(ostate, slot)
    return OS.Attestation(list(bits), OS.AttestationData(slot=slot, index=index, beacon_block_root=head, source=just, target=target), bytes(96))
