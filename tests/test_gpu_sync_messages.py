"""Sync committee messages on the GPU (b2_sync_committee_messages / _dev, Engine.sync_committee_messages / _dev, Spec.validate_sync_committee_
messages; kernels in csrc/syncmsg.cuh) against tests/sync_messages_oracle.py: every status 0-6 and every output byte of both ABI forms on the
minimal preset with real signatures, the produced SyncAggregates through b2_sync_aggregate_verify and process_sync_aggregate, three roots in
one slot, a mainnet-size slot (512 positions with repeats, every member signing through Engine.sign, 5 % bad signatures, planted duplicates)
against the oracle's closed form, the device guards, the host form's refusals and the Spec facade.
Run on an H100:
    python -m pytest tests/test_gpu_sync_messages.py -m gpu"""
import copy
import ctypes

import numpy as np
import pytest
import torch

import scenarios
import sync_messages_oracle as M
import sync_oracle as SO
from pos_evolution_b200 import spec as PS
from pos_evolution_b200._lib import B2Error
from pos_evolution_b200.engine import Engine

pytestmark = pytest.mark.gpu

N_VAL, SLOT = 64, 9
ROOT_A = scenarios._h(b"b200pos/blockroot" + SLOT.to_bytes(8, "little"))      # minimal_state's block root at SLOT
ROOT_B, ROOT_C = bytes(range(32)), bytes(range(32, 64))
GUARD_BAD_INDEX, GUARD_BAD_ROW = 1, 2
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def minimal():
    pks = scenarios.pubkeys(N_VAL)
    spec, state, cur = SO.minimal_sync_state(N_VAL, slot=SLOT, pks=pks)
    cur = list(cur)
    cur[20] = cur[12]                       # one validator on subnets 1 and 2; validator 3 holds positions 1 and 2
    state.current_sync_committee = SO.SyncCommittee([pks[v] for v in cur], SO.eth_aggregate_pubkeys([pks[v] for v in cur]))
    domain = spec.get_domain(state, PS.DOMAIN_SYNC_COMMITTEE, spec.compute_epoch_at_slot(SLOT))
    eng = Engine(0)
    eng.registry_load(np.frombuffer(b"".join(pks), np.uint8).reshape(-1, 48), np.full(N_VAL, 32 * 10**9, np.uint64))
    yield eng, spec, state, cur, pks, domain
    eng.close()


def _woff(wires):
    return np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)


def _expect_arrays(r, n, size, count=M.SUBNET_COUNT):
    """the oracle's Result as the engine's untrimmed arrays"""
    sub = size // count
    k = len(r.roots)
    cb, cs, cp = np.zeros((k, count, (sub + 7) // 8), np.uint8), np.zeros((k, count, 96), np.uint8), np.zeros((k, count), np.uint8)
    ab, asig = np.zeros((k, (size + 7) // 8), np.uint8), np.zeros((k, 96), np.uint8)
    for (j, s), c in r.contributions.items():
        cb[j, s] = np.frombuffer(M.pack(c.aggregation_bits), np.uint8)
        cs[j, s] = np.frombuffer(c.signature, np.uint8)
        cp[j, s] = 1
    for j, a in enumerate(r.aggregates):
        ab[j] = np.frombuffer(M.pack(a.sync_committee_bits), np.uint8)
        asig[j] = np.frombuffer(a.sync_committee_signature, np.uint8)
    roots = np.frombuffer(b"".join(r.roots), np.uint8).reshape(k, 32) if k else np.zeros((0, 32), np.uint8)
    return (np.array(r.status, np.int32), np.array(r.root_id, np.uint32), roots, cb, cs, cp, ab, asig)


def _assert_equal(got, want):
    names = ("status", "root_id", "roots", "contrib_bits", "contrib_sigs", "contrib_present", "agg_bits", "agg_sigs")
    for name, g, w in zip(names, got, want):
        g = np.asarray(g)
        assert g.shape == w.shape and np.array_equal(g.astype(w.dtype), w), name


def _dev(eng, wires, subnets, pv, slot, domain):
    dev = torch.device("cuda", 0)
    t = lambda a: torch.as_tensor(np.asarray(a).astype(np.int32) if np.asarray(a).dtype == np.uint32 else np.asarray(a), device=dev)  # noqa: E731
    wire = np.frombuffer(b"".join(wires), np.uint8).copy()
    r = eng.sync_committee_messages_dev(t(wire), t(_woff(wires)), t(np.asarray(subnets, np.uint32)), t(np.asarray(pv, np.uint32)), 4, slot,
                                        domain)
    torch.cuda.synchronize()
    out = [x.cpu().numpy() for x in r]
    out[1] = out[1].view(np.uint32)
    return out


def _run_both(eng, wires, subnets, pv, slot, domain):
    host = eng.sync_committee_messages(b"".join(wires), _woff(wires), subnets, pv, 4, slot, domain)
    return host, _dev(eng, wires, subnets, pv, slot, domain)


def _next_state(state, root):
    nxt = copy.deepcopy(state)
    nxt.slot = SLOT + 1
    nxt.block_roots[SLOT % len(nxt.block_roots)] = root
    return nxt


def test_minimal_every_status_both_forms(minimal):
    eng, spec, state, cur, pks, domain = minimal
    wires, subnets, expect = M.scenario(cur, domain, SLOT, [ROOT_A, ROOT_B], lambda p: int(p >= 24), N_VAL)
    want = M.validate(wires, subnets, cur, N_VAL, lambda v: pks[v], SLOT, domain)
    assert want.status == expect and set(expect) == set(range(7))
    host, dev = _run_both(eng, wires, subnets, cur, SLOT, domain)
    w = _expect_arrays(want, len(wires), 32)
    _assert_equal(host, w)
    _assert_equal(dev, w)
    assert eng.guard_flags() == 0
    # every SyncAggregate: b2_sync_aggregate_verify against the loaded committee, and process_sync_aggregate on the next slot's state
    eng.sync_committee_load(np.frombuffer(b"".join(state.current_sync_committee.pubkeys), np.uint8).reshape(-1, 48), 32)
    msgs = np.frombuffer(b"".join(M.signing_root(r, domain) for r in want.roots), np.uint8).reshape(-1, 32)
    ok = eng.sync_aggregate_verify(np.zeros(len(want.roots), np.uint32), host.agg_bits, msgs, host.agg_sigs)
    assert ok.tolist() == [1] * len(want.roots)
    for k, root in enumerate(want.roots):
        agg = SO.SyncAggregate([bool(b) for b in np.unpackbits(host.agg_bits[k], bitorder="little")[:32]], host.agg_sigs[k].tobytes())
        nxt = _next_state(state, root)
        spec.process_sync_aggregate(nxt, agg)
    # a flipped bit is refused by the same check
    bad = host.agg_bits.copy()
    bad[0, 3] ^= 1
    assert eng.sync_aggregate_verify(np.zeros(len(want.roots), np.uint32), bad, msgs, host.agg_sigs).tolist()[0] == 0


def test_three_roots(minimal):
    eng, spec, state, cur, pks, domain = minimal
    roots = [ROOT_A, ROOT_B, ROOT_C]
    wires, subnets, expect = M.scenario(cur, domain, SLOT, roots, lambda p: (p * 7 + 1) % 3, N_VAL)
    # a message list whose first accepted root is ROOT_C's: root ids follow first occurrence, not the roots' values
    order = list(range(len(wires)))
    first_c = next(a for a in order if expect[a] == M.ACCEPT and wires[a][8:40] == ROOT_C)
    order.remove(first_c)
    order.insert(0, first_c)
    wires, subnets = [wires[a] for a in order], [subnets[a] for a in order]
    want = M.validate(wires, subnets, cur, N_VAL, lambda v: pks[v], SLOT, domain)
    assert want.roots[0] == ROOT_C and len(want.roots) == 3
    few = _dev(eng, wires[:4], subnets[:4], cur, SLOT, domain)
    host, dev = _run_both(eng, wires, subnets, cur, SLOT, domain)
    w = _expect_arrays(want, len(wires), 32)
    _assert_equal(host, w)
    _assert_equal(dev, w)
    # a short list, the full one and the short one again on one engine: the same outputs as on a fresh engine
    fresh = Engine(0)
    fresh.registry_load(np.frombuffer(b"".join(pks), np.uint8).reshape(-1, 48), np.full(N_VAL, 32 * 10**9, np.uint64))
    want_few = _dev(fresh, wires[:4], subnets[:4], cur, SLOT, domain)
    fresh.close()
    _assert_equal(few, want_few)
    _assert_equal(_dev(eng, wires[:4], subnets[:4], cur, SLOT, domain), want_few)
    eng.sync_committee_load(np.frombuffer(b"".join(state.current_sync_committee.pubkeys), np.uint8).reshape(-1, 48), 32)
    msgs = np.frombuffer(b"".join(M.signing_root(r, domain) for r in want.roots), np.uint8).reshape(-1, 32)
    assert eng.sync_aggregate_verify(np.zeros(3, np.uint32), host.agg_bits, msgs, host.agg_sigs).tolist() == [1, 1, 1]


def test_mainnet_size_closed_form():
    """512 positions over 4 096 validators (secret key v + 1), with repeats inside and across subnets; every (validator, subnet) signs one
    of two roots through Engine.sign; 5 % of them sign with a wrong key first and then correctly; duplicates after accepted messages"""
    n_val, size, slot = 4096, 512, 1234567
    rng = np.random.default_rng(21)
    pv = rng.choice(n_val, size, replace=False).astype(np.uint32)
    pv[1] = pv[2] = pv[3]                          # one validator three times in subnet 0
    pv[200] = pv[300] = pv[400] = pv[100]          # one validator in all four subnets, twice in subnet 3 with position 450
    pv[450] = pv[100]
    eng = Engine(0)
    try:
        sks = [v + 1 for v in range(n_val)]
        eng.registry_load(eng.sk_to_pk(sks), np.full(n_val, 32 * 10**9, np.uint64))
        domain = bytes([7]) + bytes(range(31))
        roots = [bytes([0x11] * 32), bytes([0x22] * 32)]
        msgs = np.frombuffer(b"".join(M.signing_root(r, domain) for r in roots), np.uint8).reshape(2, 32)
        pairs = sorted({(int(pv[p]), p // 128) for p in range(size)}, key=lambda x: (x[1], x[0]))
        items = []                                 # (validator, subnet, root index, secret key)
        for v, s in pairs:
            k = int(rng.integers(0, 2))
            if rng.random() < 0.05:
                items.append((v, s, k, sks[v] + 1))
            items.append((v, s, k, sks[v]))
            if rng.random() < 0.05:
                items.append((v, s, 1 - k, sks[v]))      # a later duplicate: ignored whatever root it names
        order = rng.permutation(len(items))
        # keep each (validator, subnet)'s items in their relative order
        seq = {}
        for i in order:
            seq.setdefault(items[i][:2], []).append(i)
        for key in seq:
            seq[key].sort()
        out, taken = [], {key: 0 for key in seq}
        for i in order:
            key = items[i][:2]
            out.append(items[seq[key][taken[key]]])
            taken[key] += 1
        items = out
        sigs = eng.sign([x[3] for x in items], [x[2] for x in items], msgs)
        wires = [M.encode(slot, roots[x[2]], x[0], sigs[a].tobytes()) for a, x in enumerate(items)]
        subnets = [x[1] for x in items]
        good = {a: items[a][3] == sks[items[a][0]] for a in range(len(items))}
        want = M.validate(wires, subnets, [int(x) for x in pv], n_val, lambda v: None, slot, domain,
                          verify=lambda a, pk, m, s: good[a], secret_key=lambda v: v + 1)
        assert {0, 5, 6} <= set(want.status) and len(want.roots) == 2
        host, dev = _run_both(eng, wires, subnets, pv, slot, domain)
        w = _expect_arrays(want, len(wires), size)
        _assert_equal(host, w)
        _assert_equal(dev, w)
        # position 1, 2, 3: one validator, three bits of one contribution; the four-subnet validator in each of its contributions
        r1 = want.root_id[next(a for a in range(len(items)) if want.status[a] == 0 and items[a][:2] == (int(pv[1]), 0))]
        assert all(np.unpackbits(host.agg_bits[r1], bitorder="little")[[1, 2, 3]])
        eng.sync_committee_load(eng.sk_to_pk([sks[v] for v in pv]), size)
        assert eng.sync_aggregate_verify(np.zeros(2, np.uint32), host.agg_bits, msgs[[roots.index(bytes(x)) for x in host.roots]], host.agg_sigs).tolist() == [1, 1]
    finally:
        eng.close()


def test_device_guards(minimal):
    eng, spec, state, cur, pks, domain = minimal
    wires, subnets, expect = M.scenario(cur, domain, SLOT, [ROOT_A], lambda p: 0, N_VAL)
    eng.guard_flags()
    # a position outside the registry matches nothing: as if its validator held no position
    pv = list(cur)
    pv[30] = N_VAL + 5
    want = M.validate(wires, subnets, pv, N_VAL, lambda v: pks[v], SLOT, domain)
    dev = _dev(eng, wires, subnets, pv, SLOT, domain)
    _assert_equal(dev, _expect_arrays(want, len(wires), 32))
    assert eng.guard_flags() == GUARD_BAD_INDEX
    # a reversed woff row and one ending past the wire are status 1; the other rows are read as they are
    d = torch.device("cuda", 0)
    wire = np.frombuffer(b"".join(wires), np.uint8).copy()
    woff = _woff(wires).astype(np.int64)
    woff[3] = woff[4] + 1                           # rows 2 and 3 reversed or malformed
    woff[-1] = len(wire) + 144                      # the last row ends past the wire
    r = eng.sync_committee_messages_dev(torch.as_tensor(wire, device=d), torch.as_tensor(woff.astype(np.int32), device=d),
                                        torch.as_tensor(np.asarray(subnets, np.int32), device=d),
                                        torch.as_tensor(np.asarray(cur, np.int32), device=d), 4, SLOT, domain)
    st = r.status.cpu().numpy()
    assert st[2] == 1 and st[3] == 1 and st[-1] == 1
    assert eng.guard_flags() & GUARD_BAD_ROW


def _raw_host_call(eng, wires, woff, subnets, pv, size, count, wire_len=None):
    """b2_sync_committee_messages on sentinel-filled outputs -> (rc, outputs)"""
    n = len(woff) - 1
    sb, ab = (size // count + 7) // 8, (size + 7) // 8
    outs = [np.full(n, SENTINEL, np.int32), np.full(n, SENTINEL, np.uint32), np.full(n * 32, SENTINEL, np.uint8), np.full(1, SENTINEL, np.uint32),
            np.full(n * count * sb, SENTINEL, np.uint8), np.full(n * count * 96, SENTINEL, np.uint8), np.full(n * count, SENTINEL, np.uint8),
            np.full(n * ab, SENTINEL, np.uint8), np.full(n * 96, SENTINEL, np.uint8)]
    w = np.frombuffer(b"".join(wires), np.uint8)
    woff, sn, pvv = np.asarray(woff, np.uint32), np.asarray(subnets, np.uint32), np.asarray(pv, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)      # noqa: E731
    dom = np.zeros(32, np.uint8)
    rc = eng.lib.b2_sync_committee_messages(eng.h, p(w), len(w) if wire_len is None else wire_len, p(woff), n, p(sn), p(pvv), size, count, SLOT,
                                            p(dom), *[p(o) for o in outs])
    return rc, outs


def test_host_refusals_leave_outputs_untouched(minimal):
    eng, spec, state, cur, pks, domain = minimal
    wires = [M.encode(SLOT, ROOT_A, cur[0], bytes(96))] * 3
    woff = _woff(wires)
    rc, outs = _raw_host_call(eng, wires, woff, [0, 0, 0], cur, 32, 4)
    assert rc == 0 and outs[3][0] == 0      # a well-formed call goes through (zero signatures: status 6, no root)
    bad_cases = [
        (wires, np.array([1, 144, 288, 432], np.uint32), cur, 32, 4, None),           # woff does not start at 0
        (wires, np.array([0, 288, 144, 432], np.uint32), cur, 32, 4, None),           # woff decreases
        (wires, woff, cur, 32, 4, 431),                                                 # woff ends past the wire
        (wires, woff, list(cur[:31]) + [N_VAL], 32, 4, None),                           # a position outside the registry
        (wires, woff, list(cur[:30]), 30, 4, None),                                     # committee_size not a multiple of subnet_count
        (wires, woff, list(range(60)) * 18 + list(range(20)), 1100, 4, None),           # committee_size above 1024
    ]
    for k, (w, wo, pv, size, count, wl) in enumerate(bad_cases):
        rc, outs = _raw_host_call(eng, w, wo, [0, 0, 0], pv, size, count, wl)
        assert rc == -1, k
        assert all((o == SENTINEL).all() for o in outs), k
    fresh = Engine(0)
    try:
        rc, outs = _raw_host_call(fresh, wires, woff, [0, 0, 0], cur, 32, 4)
        assert rc == -1 and all((o == SENTINEL).all() for o in outs)      # no registry
        with pytest.raises(B2Error):
            fresh.sync_committee_messages(b"".join(wires), woff, [0, 0, 0], cur, 4, SLOT, domain)
    finally:
        fresh.close()


def test_spec_facade_matches_oracle(minimal):
    from test_gpu_sync_aggregate import _state_to_product
    eng, spec, state, cur, pks, domain = minimal
    pspec = PS.Spec(PS.MINIMAL, engine=eng)
    pstate = _state_to_product(PS, state)
    wires, subnets, expect = M.scenario(cur, domain, SLOT, [ROOT_A, ROOT_B], lambda p: int(p % 3 == 0), N_VAL)
    items = []
    for w, s in zip(wires, subnets):
        if len(w) == 144:
            items.append((s, PS.SyncCommitteeMessage(int.from_bytes(w[0:8], "little"), w[8:40], int.from_bytes(w[40:48], "little"), w[48:144])))
        else:
            items.append((s, PS.SyncCommitteeMessage(SLOT, w[8:40], int.from_bytes(w[40:48], "little"), w[48:143])))
    want = M.validate(wires, subnets, cur, N_VAL, lambda v: pks[v], SLOT, domain)
    status, contributions, aggregates = pspec.validate_sync_committee_messages(pstate, items)
    assert status == want.status
    wc = [want.contributions[k] for k in sorted(want.contributions)]
    assert [(c.slot, c.beacon_block_root, c.subcommittee_index, c.aggregation_bits, c.signature) for c in contributions] == \
        [(c.slot, c.beacon_block_root, c.subcommittee_index, c.aggregation_bits, c.signature) for c in wc]
    assert list(aggregates) == want.roots
    for k, root in enumerate(want.roots):
        assert aggregates[root].sync_committee_bits == want.aggregates[k].sync_committee_bits
        assert aggregates[root].sync_committee_signature == want.aggregates[k].sync_committee_signature
        nxt = _state_to_product(PS, _next_state(state, root))
        pspec.process_sync_aggregate(nxt, aggregates[root])
    assert aggregates[ROOT_C].sync_committee_signature == PS.G2_POINT_AT_INFINITY
    pspec.process_sync_aggregate(_state_to_product(PS, _next_state(state, ROOT_C)), aggregates[ROOT_C])      # nobody signed ROOT_C
