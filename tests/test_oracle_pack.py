"""CPU checks of the block-packing oracles (tests/pack_oracle.py): the literal global greedy equals the per-committee greedy + merge the
GPU form rests on; its gains are what the reference's process_attestation credits (oracle/spec.py) when the picks are applied in order;
and it is optimal where greedy provably is."""
import itertools

import numpy as np
import pytest

import pack_oracle as PO
import scenarios
from oracle import spec as S


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("tie_heavy", [False, True])
def test_literal_equals_per_committee(seed, tie_heavy):
    pool = PO.random_pool(seed, n_val=128 if tie_heavy else 256, comms=(4, 2) if seed % 2 else (3, 5), n_cand=80, max_out=3 + seed % 7,
                          tie_heavy=tie_heavy, bad_frac=0.1)
    lit = PO.pack_literal(pool)
    assert lit == PO.pack_per_committee(pool)
    gains = [p[3] for p in lit]
    assert all(g > 0 for g in gains)


def test_max_out_above_positive_picks_and_repeated_gains():
    pool = PO.random_pool(3, n_val=64, comms=(2, 2), n_cand=40, max_out=10**4, tie_heavy=True)
    lit = PO.pack_literal(pool)
    assert 0 < len(lit) < 10**4 and lit == PO.pack_per_committee(pool)
    # equal balances, identical rows: the same gain recurs, inside a committee and across committees
    gains = [p[3] for p in lit]
    assert len(set(gains)) < len(gains)


def test_single_bits_fold_to_one():
    pool = PO.random_pool(5, n_val=64, comms=(1, 0), n_cand=0, max_out=4)
    size = int(pool["off"][1])
    stride = pool["bits"].shape[1] if pool["bits"].size else (size + 7) // 8
    bits = np.zeros((size, stride), dtype=np.uint8)
    for j in range(size):
        bits[j, j >> 3] = 1 << (j & 7)
    pool.update(comm=np.zeros(size, dtype=np.uint32), data=np.zeros(size, dtype=np.uint32), mask=np.full(size, 7, dtype=np.uint8),
                bits=bits, ok=[True] * size)
    lit = PO.pack_literal(pool)
    assert len(lit) == 1 and lit[0][2] == (1 << size) - 1 and lit[0][4] == tuple(range(size))
    assert lit == PO.pack_per_committee(pool)


def test_greedy_is_optimal_with_one_candidate_per_committee():
    """independent committees, one folded aggregate each: the best subset of max_out is the max_out largest gains"""
    for seed in range(6):
        pool = PO.random_pool(100 + seed, n_val=64, comms=(8, 0), n_cand=0, max_out=3)
        rng = np.random.default_rng(seed)
        K = len(pool["table"])
        stride = (int(pool["off"][1]) + 7) // 8
        pool.update(comm=np.arange(K, dtype=np.uint32), data=np.arange(K, dtype=np.uint32), mask=rng.integers(1, 8, size=K).astype(np.uint8),
                    bits=rng.integers(0, 256, size=(K, stride)).astype(np.uint8), ok=[True] * K)
        lit = PO.pack_literal(pool)
        part = [list(pool["part"][0]), list(pool["part"][1])]
        gains = [PO.gain(pool, f, part) for f in PO.fold(pool)]
        best = max(sum(s) for r in range(pool["max_out"] + 1) for s in itertools.combinations(gains, r))
        assert sum(p[3] for p in lit) == best


class _AcceptAll:
    """signature checks are not what is tested here"""
    @staticmethod
    def FastAggregateVerify(pks, msg, sig):
        return True


@pytest.mark.parametrize("seed", range(4))
def test_gains_are_process_attestation_numerators(seed):
    """Pool of minimal-preset attestations (two epochs, several votes per committee, aggregates and single bits): applying the picks in
    order with the reference's process_attestation sets exactly the flags each gain counts, and credits the proposer sum(gain // 1024)."""
    rng = np.random.default_rng(seed)
    _, state = scenarios.minimal_state(64, slot=17 + seed)
    spec = S.Spec(S.MINIMAL, bls_module=_AcceptAll)
    state.current_epoch_participation = [int(x) for x in (rng.integers(0, 8, size=64) * (rng.random(64) < 0.3))]
    state.previous_epoch_participation = [int(x) for x in (rng.integers(0, 8, size=64) * (rng.random(64) < 0.3))]
    cur = spec.get_current_epoch(state)
    pool = []
    for slot in range(max(0, state.slot - 8), state.slot):
        if spec.compute_epoch_at_slot(slot) not in (cur, cur - 1):
            continue
        for index in range(spec.get_committee_count_per_slot(state, spec.compute_epoch_at_slot(slot))):
            n = len(spec.get_beacon_committee(state, slot, index))
            epoch = spec.compute_epoch_at_slot(slot)
            just = state.current_justified_checkpoint if epoch == cur else state.previous_justified_checkpoint
            target = S.Checkpoint(epoch, spec.get_block_root(state, epoch) if spec.compute_start_slot_at_epoch(epoch) < state.slot else b"t" * 32)
            for head in (spec.get_block_root_at_slot(state, slot), b"\x11" * 32):
                data = S.AttestationData(slot=slot, index=index, beacon_block_root=head, source=just, target=target)
                for _ in range(int(rng.integers(1, 4))):
                    pool.append(S.Attestation([bool(b) for b in (rng.random(n) < rng.choice([0.3, 0.7]))], data, bytes(96)))
                j = int(rng.integers(0, n))
                pool.append(S.Attestation([i == j for i in range(n)], data, bytes(96)))
    # the pack_oracle form of the pool, as Spec.get_attestations_for_block builds it
    committees, data_ids, datas = {}, {}, []
    members, off, table, comm, data, mask, rows = [], [0], [], [], [], [], []
    for att in pool:
        d = att.data
        committee = spec.get_beacon_committee(state, d.slot, d.index)
        flags = spec.get_attestation_participation_flag_indices(state, d, state.slot - d.slot)
        if (d.slot, d.index) not in committees:
            committees[(d.slot, d.index)] = len(table)
            members += committee
            off.append(len(members))
            table.append(0 if d.target.epoch == cur else 1)
        root = S.hash_tree_root_attestation_data(d)
        if root not in data_ids:
            data_ids[root] = len(datas)
            datas.append(d)
        comm.append(committees[(d.slot, d.index)])
        data.append(data_ids[root])
        mask.append(sum(1 << f for f in flags))
        rows.append(att.aggregation_bits)
    stride = (max(len(r) for r in rows) + 7) // 8
    bits = np.zeros((len(rows), stride), dtype=np.uint8)
    for c, r in enumerate(rows):
        packed = np.packbits(np.asarray(r, dtype=np.uint8), bitorder="little")
        bits[c, :len(packed)] = packed
    per_inc = spec.get_base_reward_per_increment(state)
    opool = {"members": members, "off": off, "table": table, "comm": comm, "data": data, "mask": mask, "bits": bits, "ok": [True] * len(rows),
             "eff": [v.effective_balance for v in state.validators], "part": (list(state.current_epoch_participation), list(state.previous_epoch_participation)),
             "inc": S.MINIMAL.EFFECTIVE_BALANCE_INCREMENT, "per_inc": per_inc, "max_out": 6}
    picks = PO.pack_literal(opool)
    assert picks == PO.pack_per_committee(opool) and len(picks) > 0
    proposer = spec.get_beacon_proposer_index(state)
    bal0 = state.balances[proposer]
    denominator = (S.WEIGHT_DENOMINATOR - S.PROPOSER_WEIGHT) * S.WEIGHT_DENOMINATOR // S.PROPOSER_WEIGHT
    for k, d, row, g, _ in picks:
        n = off[k + 1] - off[k]
        att = S.Attestation([bool((row >> j) & 1) for j in range(n)], datas[d], bytes(96))
        before = (list(state.current_epoch_participation), list(state.previous_epoch_participation))
        spec.process_attestation(state, att)
        credited = 0
        for t, (old, new) in enumerate(zip(before, (state.current_epoch_participation, state.previous_epoch_participation))):
            for v in range(64):
                for f in range(3):
                    if (new[v] >> f) & 1 and not (old[v] >> f) & 1:
                        credited += spec.get_base_reward(state, v) * S.PARTICIPATION_FLAG_WEIGHTS[f]
        assert credited == g
    assert state.balances[proposer] - bal0 == sum(g // denominator for _, _, _, g, _ in picks)


def test_preset_max_attestations():
    from pos_evolution_b200 import spec as GS
    assert GS.MAINNET.MAX_ATTESTATIONS == GS.MINIMAL.MAX_ATTESTATIONS == 128
