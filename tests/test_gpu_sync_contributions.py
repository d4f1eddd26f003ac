"""Sync committee contributions on the GPU (b2_sync_contribution_and_proof_intake / _dev, Engine.sync_contribution_and_proof_intake / _dev,
Spec.validate_sync_contribution_and_proofs; kernels in csrc/synccontrib.cuh) against tests/sync_contributions_oracle.py: every status 0-12 and
every output byte of both ABI forms on the minimal preset with real signatures and three roots, the produced SyncAggregates through
b2_sync_aggregate_verify and process_sync_aggregate, a mainnet-size slot against closed-form sums, a 4 096-item worst-case list, the device
guards, the host form's refusals, the RLC verify mode and the Spec facade.
Run on an H100:
    python -m pytest tests/test_gpu_sync_contributions.py -m gpu -s"""
import copy
import ctypes
import statistics
import time

import numpy as np
import pytest
import torch

import scenarios
import sync_contributions_oracle as C
import sync_oracle as SO
from oracle import bls_sig as B
from oracle.bls12_381 import R
from pos_evolution_b200 import spec as PS
from pos_evolution_b200._lib import B2Error
from pos_evolution_b200.engine import Engine

pytestmark = pytest.mark.gpu

N_VAL, SLOT = 64, 9
ROOT_A = scenarios._h(b"b200pos/blockroot" + SLOT.to_bytes(8, "little"))      # minimal_state's block root at SLOT
ROOT_B, ROOT_C = bytes(range(32)), bytes(range(32, 64))
GUARD_BAD_INDEX, GUARD_BAD_ROW = 1, 2
SENTINEL = 0xA5
NEED = {0: 1, 1: 2, 2: 2, 3: 1}


def _domains(spec, state, slot):
    e = spec.compute_epoch_at_slot(slot)
    return b"".join(spec.get_domain(state, d, e) for d in (PS.DOMAIN_SYNC_COMMITTEE, PS.DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF,
                                                           PS.DOMAIN_CONTRIBUTION_AND_PROOF))


@pytest.fixture(scope="module")
def minimal():
    pks = scenarios.pubkeys(N_VAL)
    spec, state, cur = SO.minimal_sync_state(N_VAL, slot=SLOT, pks=pks)
    domains = _domains(spec, state, SLOT)
    # aggregators selected at target 1 on every subnet; validator 3 keeps positions 1 and 2
    pv = C.with_aggregators(cur, N_VAL, lambda p: C.Signer(p, domains, SLOT), 1, NEED)
    assert pv[1] == pv[2] == 3
    state.current_sync_committee = SO.SyncCommittee([pks[v] for v in pv], SO.eth_aggregate_pubkeys([pks[v] for v in pv]))
    eng = Engine(0)
    eng.registry_load(np.frombuffer(b"".join(pks), np.uint8).reshape(-1, 48), np.full(N_VAL, 32 * 10**9, np.uint64))
    yield eng, spec, state, pv, pks, domains
    eng.close()


def _woff(wires):
    return np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32)


def _assert_equal(got, want):
    for name, g, w in zip(("status", "root_id", "roots", "best", "agg_bits", "agg_sigs"), got, want):
        g = np.asarray(g)
        assert g.shape == w.shape and np.array_equal(g.astype(w.dtype), w), name


def _dev(eng, wires, pv, slot, domains, target):
    dev = torch.device("cuda", 0)
    t = lambda a: torch.as_tensor(np.asarray(a).astype(np.int32) if np.asarray(a).dtype == np.uint32 else np.asarray(a), device=dev)  # noqa: E731
    wire = np.frombuffer(b"".join(wires), np.uint8).copy()
    r = eng.sync_contribution_and_proof_intake_dev(t(wire), t(_woff(wires)), t(np.asarray(pv, np.uint32)), 4, slot, domains, target)
    torch.cuda.synchronize()
    out = [x.cpu().numpy() for x in r]
    out[1], out[3] = out[1].view(np.uint32), out[3].view(np.uint32)
    return out


def _run_both(eng, wires, pv, slot, domains, target):
    host = eng.sync_contribution_and_proof_intake(b"".join(wires), _woff(wires), pv, 4, slot, domains, target)
    return host, _dev(eng, wires, pv, slot, domains, target)


def _scenario(pv, domains, roots):
    sg = C.Signer(pv, domains, SLOT)
    wires, expect = C.scenario(sg, roots, 1, N_VAL)
    on = lambda *ix: [i in ix for i in range(sg.sub)]      # noqa: E731
    wires.append(sg.item(pv[0], 0, roots[-1], on(0, 1, 2)))      # validator 3 at positions 1 and 2: its key counts twice
    expect.append(C.ACCEPT)
    return wires, expect


def _next_state(state, root):
    nxt = copy.deepcopy(state)
    nxt.slot = SLOT + 1
    nxt.block_roots[SLOT % len(nxt.block_roots)] = root
    return nxt


def _verify_aggregates(eng, spec, state, domains, roots, agg_bits, agg_sigs):
    eng.sync_committee_load(np.frombuffer(b"".join(state.current_sync_committee.pubkeys), np.uint8).reshape(-1, 48), 32)
    msgs = np.frombuffer(b"".join(C.signing_root(r, domains[:32]) for r in roots), np.uint8).reshape(-1, 32)
    assert eng.sync_aggregate_verify(np.zeros(len(roots), np.uint32), agg_bits, msgs, agg_sigs).tolist() == [1] * len(roots)
    for k, root in enumerate(roots):
        agg = SO.SyncAggregate([bool(b) for b in np.unpackbits(agg_bits[k], bitorder="little")[:32]], agg_sigs[k].tobytes())
        spec.process_sync_aggregate(_next_state(state, root), agg)


def test_minimal_every_status_both_forms(minimal):
    eng, spec, state, pv, pks, domains = minimal
    wires, expect = _scenario(pv, domains, [ROOT_A, ROOT_B, ROOT_C])
    want = C.validate(wires, pv, N_VAL, lambda v: pks[v], SLOT, domains, target=1)
    assert want.status == expect and set(expect) == set(range(13)) and len(want.roots) == 3
    w = C.expect_arrays(want, size=32)
    few = _dev(eng, wires[:5], pv, SLOT, domains, 1)
    host, dev = _run_both(eng, wires, pv, SLOT, domains, 1)
    _assert_equal(host, w)
    _assert_equal(dev, w)
    # a short list, the full one, the short one again: the grown scratch gives the oracle's outputs
    _assert_equal(few, C.expect_arrays(C.validate(wires[:5], pv, N_VAL, lambda v: pks[v], SLOT, domains, target=1), size=32))
    _assert_equal(_dev(eng, wires[:5], pv, SLOT, domains, 1), few)
    assert eng.guard_flags() == 0
    _verify_aggregates(eng, spec, state, domains, want.roots, host.agg_bits, host.agg_sigs)
    # the RLC verify mode gives the same outputs
    eng.set_verify_mode(True, bytes(range(32)))
    try:
        _assert_equal(eng.sync_contribution_and_proof_intake(b"".join(wires), _woff(wires), pv, 4, SLOT, domains, 1), w)
        _assert_equal(_dev(eng, wires, pv, SLOT, domains, 1), w)
    finally:
        eng.set_verify_mode(False)


def test_device_guards(minimal):
    eng, spec, state, pv, pks, domains = minimal
    wires, expect = _scenario(pv, domains, [ROOT_A, ROOT_B, ROOT_C])
    eng.guard_flags()
    bad = list(pv)
    bad[25] = N_VAL + 5      # covered by subnet 3's accepted item: it now fails FastAggregateVerify
    pk = lambda v: pks[v] if v < N_VAL else None      # noqa: E731
    want = C.validate(wires, bad, N_VAL, pk, SLOT, domains, target=1,
                      fast_verify=lambda a, keys, m, s: None not in keys and B.FastAggregateVerify(keys, m, s))
    a3 = next(a for a, w in enumerate(wires) if expect[a] == C.ACCEPT and C.decode(w, 1)[3] == 3)
    assert want.status[a3] == C.BAD_CONTRIBUTION
    _assert_equal(_dev(eng, wires, bad, SLOT, domains, 1), C.expect_arrays(want, size=32))
    assert eng.guard_flags() == GUARD_BAD_INDEX
    d = torch.device("cuda", 0)
    wire = np.frombuffer(b"".join(wires), np.uint8).copy()
    woff = _woff(wires).astype(np.int64)
    woff[3] = woff[4] + 1                           # rows 2 and 3 reversed or malformed
    woff[-1] = len(wire) + 345                      # the last row ends past the wire
    r = eng.sync_contribution_and_proof_intake_dev(torch.as_tensor(wire, device=d), torch.as_tensor(woff.astype(np.int32), device=d),
                                                   torch.as_tensor(np.asarray(pv, np.int32), device=d), 4, SLOT, domains, 1)
    st = r.status.cpu().numpy()
    assert st[2] == 1 and st[3] == 1 and st[-1] == 1
    assert eng.guard_flags() & GUARD_BAD_ROW


def _raw_host_call(eng, wires, woff, pv, size, count, target=16, wire_len=None):
    """b2_sync_contribution_and_proof_intake on sentinel-filled outputs -> (rc, outputs)"""
    n = len(woff) - 1
    outs = [np.full(n, SENTINEL, np.int32), np.full(n, SENTINEL, np.uint32), np.full(n * 32, SENTINEL, np.uint8), np.full(1, SENTINEL, np.uint32),
            np.full(n * count, SENTINEL, np.uint32), np.full(n * ((size + 7) // 8), SENTINEL, np.uint8), np.full(n * 96, SENTINEL, np.uint8)]
    w = np.frombuffer(b"".join(wires), np.uint8)
    woff, pvv = np.asarray(woff, np.uint32), np.asarray(pv, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)      # noqa: E731
    dom = np.zeros(96, np.uint8)
    rc = eng.lib.b2_sync_contribution_and_proof_intake(eng.h, p(w), len(w) if wire_len is None else wire_len, p(woff), n, p(pvv), size, count,
                                                       SLOT, p(dom), target, *[p(o) for o in outs])
    return rc, outs


def test_host_refusals_leave_outputs_untouched(minimal):
    eng, spec, state, pv, pks, domains = minimal
    wires = [C.encode(pv[8], SLOT, ROOT_A, 1, [True] * 8, bytes(96), bytes(96), bytes(96))] * 3
    woff = _woff(wires)
    rc, outs = _raw_host_call(eng, wires, woff, pv, 32, 4)
    assert rc == 0 and outs[3][0] == 0      # a well-formed call goes through (zero signatures: status 10, no root)
    bad_cases = [
        (np.array([1, 345, 690, 1035], np.uint32), pv, 32, 4, 16, None),           # woff does not start at 0
        (np.array([0, 690, 345, 1035], np.uint32), pv, 32, 4, 16, None),           # woff decreases
        (woff, pv, 32, 4, 16, 1034),                                                 # woff ends past the wire
        (woff, list(pv[:31]) + [N_VAL], 32, 4, 16, None),                            # a position outside the registry
        (woff, list(pv[:30]), 30, 4, 16, None),                                      # committee_size not a multiple of subnet_count
        (woff, list(range(60)) * 18 + list(range(20)), 1100, 4, 16, None),           # committee_size above 1024
        (woff, pv, 32, 4, 0, None),                                                  # target_aggregators == 0
        (np.array([0], np.uint32), pv, 32, 4, 16, None),                             # n == 0
    ]
    for k, (wo, p, size, count, target, wl) in enumerate(bad_cases):
        rc, outs = _raw_host_call(eng, wires, wo, p, size, count, target, wl)
        assert rc == -1, k
        assert all((o == SENTINEL).all() for o in outs), k
    fresh = Engine(0)
    try:
        rc, outs = _raw_host_call(fresh, wires, woff, pv, 32, 4)
        assert rc == -1 and all((o == SENTINEL).all() for o in outs)      # no registry
        with pytest.raises(B2Error):
            fresh.sync_contribution_and_proof_intake(b"".join(wires), woff, pv, 4, SLOT, domains)
    finally:
        fresh.close()


def _product_items(wires, sb=1):
    out = []
    for w in wires:
        g, slot, root, s, row, sig, proof, outer = C.decode(w, sb)
        bits = [bool(row[0] >> i & 1) for i in range(8)]
        out.append(PS.SignedContributionAndProof(PS.ContributionAndProof(g, PS.SyncCommitteeContribution(slot, root, s, bits, sig), proof), outer))
    return out


def test_spec_facade_matches_oracle(minimal):
    from test_gpu_sync_aggregate import _state_to_product
    eng, spec, state, pv, pks, domains = minimal
    pspec = PS.Spec(PS.MINIMAL, engine=eng)
    wires, expect = _scenario(pv, domains, [ROOT_A, ROOT_B])
    wires = [w for w in wires if len(w) == 345]
    want = C.validate(wires, pv, N_VAL, lambda v: pks[v], SLOT, domains, target=16)      # the preset's target: every member selects itself
    status, aggregates = pspec.validate_sync_contribution_and_proofs(_state_to_product(PS, state), _product_items(wires))
    assert status == want.status
    assert list(aggregates) == want.roots
    for k, root in enumerate(want.roots):
        assert aggregates[root].sync_committee_bits == want.aggregates[k].sync_committee_bits
        assert aggregates[root].sync_committee_signature == want.aggregates[k].sync_committee_signature
        pspec.process_sync_aggregate(_state_to_product(PS, _next_state(state, root)), aggregates[root])
    assert aggregates[ROOT_C].sync_committee_signature == PS.G2_POINT_AT_INFINITY      # no contribution for ROOT_C
    # at a period boundary (state.slot + 1 starts the next period) the next committee is the one checked
    b = copy.deepcopy(state)
    b.slot = PS.MINIMAL.SLOTS_PER_EPOCH * PS.MINIMAL.EPOCHS_PER_SYNC_COMMITTEE_PERIOD - 1
    nxt = [pks.index(pk) for pk in b.next_sync_committee.pubkeys]
    dom_b = _domains(spec, b, b.slot)
    sg = C.Signer(nxt, dom_b, b.slot)
    on = lambda *ix: [i in ix for i in range(8)]      # noqa: E731
    outsider = next(v for v in pv[8:16] if v not in nxt[8:16])      # in the current committee's subnet 1, not the next one's
    items = [sg.item(nxt[8], 1, ROOT_B, on(0, 1, 2)), sg.item(outsider, 1, ROOT_B, on(3)), sg.item(nxt[16], 2, ROOT_B, on(0, 5))]
    want = C.validate(items, nxt, N_VAL, lambda v: pks[v], b.slot, dom_b, target=16)
    assert want.status == [C.ACCEPT, C.NOT_IN_SUBNET, C.ACCEPT]
    status, aggregates = pspec.validate_sync_contribution_and_proofs(_state_to_product(PS, b), _product_items(items))
    assert status == want.status
    assert aggregates[ROOT_B].sync_committee_signature == want.aggregates[0].sync_committee_signature


def _signed_batch(eng, sks, msgs):
    """Engine.sign of one message per key"""
    m = np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32)
    return [bytes(x) for x in eng.sign([k % R for k in sks], np.arange(len(msgs), dtype=np.uint32), m)]


def _build_items(eng, plan, pv, sk, domains, slot, sub):
    """plan: [(aggregator, subnet, root, bit list, (proof ok, outer ok, contribution ok))] -> wires, signed through Engine.sign in three
    batches: selection proofs and contribution signatures, then the outer signatures over the ContributionAndProof roots"""
    n = len(plan)
    proofs = _signed_batch(eng, [sk(g) + (0 if ok[0] else 1) for g, s, r, b, ok in plan],
                           [C.signing_root(C.selection_data_root(slot, s), domains[32:64]) for g, s, r, b, ok in plan])
    sigs = _signed_batch(eng, [sum(sk(pv[s * sub + i]) for i, x in enumerate(b) if x) + (0 if ok[2] else 1) for g, s, r, b, ok in plan],
                         [C.signing_root(r, domains[:32]) for g, s, r, b, ok in plan])
    caps = [C.signing_root(C.contribution_and_proof_root(g, slot, r, s, C.pack(b), sigs[a], proofs[a]), domains[64:96])
            for a, (g, s, r, b, ok) in enumerate(plan)]
    outers = _signed_batch(eng, [sk(g) + (0 if ok[1] else 1) for g, s, r, b, ok in plan], caps)
    return [C.encode(g, slot, r, s, b, sigs[a], proofs[a], outers[a]) for a, (g, s, r, b, ok) in enumerate(plan)][:n]


def test_mainnet_size_closed_form():
    """512 positions over 4 096 validators (secret key v + 1) with repeats inside and across subnets; 16 selected aggregators per subnet
    (the preset's target) on two roots; planted subsets, equal-bits duplicates, second roots, 5 % bad signatures"""
    n_val, size, slot, sub = 4096, 512, 1234567, 128
    rng = np.random.default_rng(31)
    pv = rng.choice(n_val, size, replace=False).astype(np.uint32)
    pv[1] = pv[2] = pv[3]
    pv[200] = pv[300] = pv[400] = pv[100]
    pv[450] = pv[100]
    sk = lambda v: int(v) + 1      # noqa: E731
    eng = Engine(0)
    try:
        eng.registry_load(eng.sk_to_pk([sk(v) for v in range(n_val)]), np.full(n_val, 32 * 10**9, np.uint64))
        domains = bytes([7]) + bytes(range(31)) + bytes([8]) + bytes(range(31)) + bytes([9]) + bytes(range(31))
        roots = [bytes([0x11] * 32), bytes([0x22] * 32)]
        pairs = sorted({(int(pv[p]), p // sub) for p in range(size)})
        proofs = _signed_batch(eng, [sk(v) for v, s in pairs], [C.signing_root(C.selection_data_root(slot, s), domains[32:64]) for v, s in pairs])
        chosen = {s: [] for s in range(4)}
        for (v, s), p in zip(pairs, proofs):
            if C.is_aggregator(p, sub, 16) and len(chosen[s]) < 16:
                chosen[s].append(v)
        assert all(len(chosen[s]) >= 8 for s in range(4)), {s: len(x) for s, x in chosen.items()}
        plan = []
        for s in range(4):
            for j, v in enumerate(chosen[s]):
                bits = [bool(x) for x in rng.random(sub) < 0.5]
                ok = tuple(bool(x) for x in rng.random(3) >= 0.05 / 3)
                plan.append((v, s, roots[j % 2], bits, ok))
                if j % 5 == 1:
                    plan.append((chosen[s][j - 1], s, roots[(j - 1) % 2], bits, (True, True, True)))   # the same aggregator: 8 or 9
                if j % 7 == 3:
                    plan.append((v, s, roots[j % 2], bits, (True, True, True)))                        # an equal-bits duplicate
                if j % 4 == 2:
                    sub_bits = [x and rng.random() < 0.5 for x in bits]
                    plan.append((chosen[s][(j + 1) % len(chosen[s])], s, roots[j % 2], sub_bits if any(sub_bits) else bits, (True, True, True)))
        order = rng.permutation(len(plan))
        plan = [plan[i] for i in order]
        wires = _build_items(eng, plan, pv, sk, domains, slot, sub)
        flags = [p[4] for p in plan]
        want = C.validate(wires, [int(x) for x in pv], n_val, lambda v: None, slot, domains, target=16,
                          verify=lambda a, pk, m, s, which: flags[a][which], fast_verify=lambda a, keys, m, s: flags[a][2])
        assert {0, 8, 9} <= set(want.status) and len(want.roots) == 2
        host, dev = _run_both(eng, wires, pv, slot, domains, 16)
        w = C.expect_arrays(want, size=size)
        _assert_equal(host, w)
        _assert_equal(dev, w)
        # closed form: each root's aggregate is Sign(sum of the secret keys of its set positions, with multiplicity)
        for k, root in enumerate(want.roots):
            bits = np.unpackbits(host.agg_bits[k], bitorder="little")[:size]
            assert host.agg_sigs[k].tobytes() == _signed_batch(eng, [sum(sk(pv[p]) for p in range(size) if bits[p])],
                                                               [C.signing_root(root, domains[:32])])[0]
        eng.sync_committee_load(eng.sk_to_pk([sk(v) for v in pv]), size)
        msgs = np.frombuffer(b"".join(C.signing_root(r, domains[:32]) for r in want.roots), np.uint8).reshape(-1, 32)
        assert eng.sync_aggregate_verify(np.zeros(2, np.uint32), host.agg_bits, msgs, host.agg_sigs).tolist() == [1, 1]
    finally:
        eng.close()


def test_worst_case_list():
    """4 096 items on one subnet and root, every one past checks 1-7 (target = sub: every proof selects), honest signatures over random
    bit rows: the list-order pass compares each item with up to 128 accepted ones.  Prints the wall time per call."""
    n_val, size, slot, sub, n = 1024, 512, 777, 128, 4096
    rng = np.random.default_rng(41)
    pv = rng.choice(n_val, size, replace=False).astype(np.uint32)
    sk = lambda v: int(v) * 3 + 7      # noqa: E731
    eng = Engine(0)
    try:
        eng.registry_load(eng.sk_to_pk([sk(v) for v in range(n_val)]), np.full(n_val, 32 * 10**9, np.uint64))
        domains = bytes(range(96))
        root = bytes([0x33] * 32)
        plan = []
        for a in range(n):
            bits = [bool(x) for x in rng.random(sub) < rng.uniform(0.05, 0.95)]
            bits[int(rng.integers(0, sub))] = True
            plan.append((int(pv[int(rng.integers(0, sub))]), 0, root, bits, (True, True, True)))
        wires = _build_items(eng, plan, pv, sk, domains, slot, sub)
        want = C.validate(wires, [int(x) for x in pv], n_val, lambda v: None, slot, domains, target=sub,
                          verify=lambda a, pk, m, s, which: True, fast_verify=lambda a, keys, m, s: True)
        assert want.status.count(C.ACCEPT) > 1 and set(want.status) <= {0, 8, 9}
        blob, woff = b"".join(wires), _woff(wires)
        host = eng.sync_contribution_and_proof_intake(blob, woff, pv, 4, slot, domains, sub)
        _assert_equal(host, C.expect_arrays(want, size=size))
        times = []
        for _ in range(3):
            t0 = time.perf_counter()
            eng.sync_contribution_and_proof_intake(blob, woff, pv, 4, slot, domains, sub)
            times.append(time.perf_counter() - t0)
        print("\nworst-case list: %d items on one (root, subnet), %d accepted: %.2f ms per call (median of 3, wall, host form) on %s"
              % (n, want.status.count(0), 1e3 * statistics.median(times), torch.cuda.get_device_name(0)))
    finally:
        eng.close()
