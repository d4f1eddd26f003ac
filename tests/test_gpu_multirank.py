"""Strong scaling: ONE 2^20-validator epoch sharded by slot over the ranks (BASELINE.json configs 4/5, SURVEY.md section 8e), every
rank a process with its own context.

Every rank runs the sharded EpochProcessor (pipelined form, several epochs, tampered signatures on every rank) and reports what it saw;
the parent process compares EVERY rank with the single-process oracle:
  * the all-gathered verdict vector of every epoch == the expected one (exactly the tampered committees rejected);
  * the all-gathered aggregate signatures == oracle.Sign(sum of the committee's secret keys, message) on a sample from each rank's share;
  * the replicated latest-message table after the last epoch == the sequential update_latest_messages of the numpy oracle;
  * the head of every epoch (vote scatter of N/world validators per rank -> all-reduce -> head) == the numpy oracle's get_head;
  * EpochProcessor.get_head (the path bench.py times at N > 1) == the same head in its three-stage form (scatter, all-reduce, tree) and,
    per_device only, in the one-kernel form with the all-reduce fused in over NVLink peer memory (b2_get_head_multi), repeatedly.

Two layouts (tests/rank_group.py): per_device, world 2 with one GPU per rank over NCCL (skipped below 2 GPUs); shared_device, the ranks
sharing one GPU over host-staged gloo, at world 2 and 4.  The shared layout runs every device call of the sharded epoch but not NCCL,
NVLink, the fused get_head across ranks or any multi-GPU timing."""
import hashlib

import numpy as np
import pytest

import rank_group

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

N_EPOCHS = 3


def _plan(bench):
    """target epochs / voted blocks of the epochs and the tampered committees (two per rank at world 2, one at world 4)"""
    te = [np.full(bench.N_AGG, 7 + k, dtype=np.int64) for k in range(N_EPOCHS)]
    base = (bench.N_BLOCKS - 1 - (np.arange(bench.N_AGG) % 64)).astype(np.int64)
    bk = [((base - 97 * k) % bench.N_BLOCKS).astype(np.int32) for k in range(N_EPOCHS)]
    bad = [5, 700, 1500, 2047]
    return te, bk, bad


def _worker(rank, world, port, q, shared):
    import torch.distributed as dist
    import bench
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    dev = rank_group.init(rank, world, port, shared)
    eng = Engine(dev.index)
    W = bench.build_world(eng, rank, np, PS, shard=(rank, world))
    ep = EpochProcessor(eng, bench.N_AGG, bench.N_VAL, bench.COMMITTEE_SIZE // 8, bench.N_BLOCKS, process_group=dist.group.WORLD, device=dev,
                        depth=4, shard=(rank, world), n_validators=bench.N_VAL)
    ep.set_committees(W["members"], W["off"])
    te, bk, bad = _plan(bench)
    sigs = W["sigs"].copy()                       # this rank's rows [m0, m1) of the epoch's signatures
    for a in bad:
        if ep.a0 <= a < ep.a1:                    # a valid signature of ANOTHER message: only the pairing can tell
            other = ep.a0 + (a - ep.a0 + 1) % ep.n_loc
            sigs[int(W["off"][a]) - ep.m0 + 3] = W["sigs"][int(W["off"][other]) - ep.m0 + 9]
    d_sigs = torch.as_tensor(sigs, device=dev)
    d_bits = torch.full((bench.N_AGG, bench.COMMITTEE_SIZE // 8), 0xFF, dtype=torch.uint8, device=dev)
    d_msgs = torch.as_tensor(W["msgs"], device=dev)
    keep, out = [], []
    for k in range(N_EPOCHS):
        dk = (torch.as_tensor(te[k], device=dev), torch.as_tensor(bk[k], device=dev))
        keep.append(dk)
        t = ep.submit_dev(d_sigs, d_bits, d_msgs, dk[0], dk[1], 0, bench.N_BLOCKS - 1, W["boost"], last=(k == N_EPOCHS - 1))
        if t is not None:
            out.append(t)
    out += ep.drain()
    res = []
    for t in out:
        ok, head = t.wait()
        res.append((ok.cpu().numpy().tobytes(), head))
    agg = out[-1].aggregate_signatures().cpu().numpy()
    e, b, h = eng.latest_messages_read()
    lmd = hashlib.sha256(e[h == 1].tobytes() + b[h == 1].tobytes() + h.tobytes()).hexdigest()
    head_again = ep.get_head(0, bench.N_BLOCKS - 1, W["boost"])                       # scatter kernel -> all-reduce -> tree kernel
    torch.cuda.synchronize()
    if shared:
        # The fused kernel spins on flags its peers raise over NVLink: ranks time-slicing one GPU could leave it waiting for a peer
        # that cannot run, so it is only run with a GPU per rank.
        heads_fused = None
        head_no_boost = ep.get_head(0, -1, 0, fused=False)
    else:
        assert ep.enable_fused_get_head(), ep.fused_head_error                            # CUDA IPC exchange blocks over NVLink
        heads_fused = [ep.get_head(0, bench.N_BLOCKS - 1, W["boost"], fused=True) for _ in range(5)]   # one kernel per rank, all-reduce fused in
        heads_fused.append(ep.get_head(0, -1, 0, fused=True))
        head_no_boost = ep.get_head(0, -1, 0, fused=False)
    sample = [a for a in (0, 511, 1023, 1024, 1100, 2046) if a not in bad]
    q.put((rank, res, {a: bytes(agg[a]) for a in sample}, lmd, head_again, eng.guard_flags(), heads_fused, head_no_boost))
    dist.barrier()
    dist.destroy_process_group()
    eng.close()


@pytest.mark.parametrize("layout,world", [("per_device", 2), ("shared_device", 2), ("shared_device", 4)])
def test_sharded_epoch_equals_the_oracle(layout, world):
    import bench
    from oracle import bls_sig as B
    from oracle import fast
    if layout == "per_device" and torch.cuda.device_count() < world:
        pytest.skip("needs >= %d GPUs" % world)
    results = rank_group.run(_worker, world, args=(layout == "shared_device",))

    # ---- the single-process oracle of the same three epochs
    class _Null:       # build the (deterministic) world arrays without a GPU: only what the oracle needs
        pass
    te, bk, bad = _plan(bench)
    sk0 = int.from_bytes(hashlib.sha256(b"b200pos/sk0").digest(), "big") % (bench.R_ORDER >> 1) or 1
    delta = int.from_bytes(hashlib.sha256(b"b200pos/skd").digest(), "big") >> 64
    seed = hashlib.sha256(b"b200pos/epoch-seed" + (0).to_bytes(8, "little")).digest()
    members = fast.shuffle_permutation(bench.N_VAL, seed, 90)
    off = (np.arange(bench.N_AGG + 1, dtype=np.uint64) * bench.COMMITTEE_SIZE).astype(np.uint32)
    msgs = [hashlib.sha256(b"b200pos/signing-root" + (0).to_bytes(4, "little") + a.to_bytes(4, "little")).digest() for a in range(bench.N_AGG)]
    Wo = dict(members=members, off=off, sk0=sk0, delta=delta)
    rng = np.random.default_rng(4)
    eff = np.where(rng.random(bench.N_VAL) < 0.9, 32, rng.integers(16, 33, size=bench.N_VAL)).astype(np.uint64) * np.uint64(10**9)
    active = np.ones(bench.N_VAL, dtype=np.uint8)
    trng = np.random.default_rng(4)
    parent = np.zeros(bench.N_BLOCKS, dtype=np.uint32)
    back = trng.geometric(0.7, size=bench.N_BLOCKS) - 1
    trng.binomial(2, 0.1, size=bench.N_BLOCKS)
    for i in range(1, bench.N_BLOCKS):
        parent[i] = max(0, i - 1 - int(back[i]))
    roots = np.frombuffer(b"".join(hashlib.sha256(i.to_bytes(8, "little")).digest() for i in range(bench.N_BLOCKS)), dtype=np.uint8).reshape(-1, 32)
    leaf_viable = (trng.random(bench.N_BLOCKS) >= 0.05).astype(np.uint8)
    msg_block = (bench.N_BLOCKS - 1 - np.minimum(bench.N_BLOCKS - 1, rng.geometric(0.002, size=bench.N_VAL))).astype(np.uint32)
    has_msg = (rng.random(bench.N_VAL) >= 0.01).astype(np.uint8)
    equiv = (rng.random(bench.N_VAL) < 0.001).astype(np.uint8)
    boost = (bench.N_VAL // 32) * (int(eff.astype(object).sum()) // bench.N_VAL) * 40 // 100
    expect_ok = np.ones(bench.N_AGG, dtype=np.uint8)
    expect_ok[bad] = 0
    m_epoch = np.ones(bench.N_VAL, dtype=np.uint64)
    want_heads = []
    keep = fast.ghost_viable(parent, leaf_viable)
    for k in range(N_EPOCHS):
        for a in np.nonzero(expect_ok)[0]:
            fast.lmd_update(m_epoch, msg_block, has_msg, equiv, members[off[a]:off[a + 1]], int(te[k][a]), int(bk[k][a]))
        w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, bench.N_BLOCKS - 1, boost)
        want_heads.append(fast.ghost_head(parent, roots, keep, w, 0))
    want_lmd = hashlib.sha256(m_epoch[has_msg == 1].tobytes() + msg_block[has_msg == 1].tobytes() + has_msg.tobytes()).hexdigest()

    w_nb = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, -1, 0)
    want_no_boost = fast.ghost_head(parent, roots, keep, w_nb, 0)
    for rank, res, agg_sample, lmd, head_again, guard, heads_fused, head_no_boost in results:
        if heads_fused is not None:
            assert heads_fused == [want_heads[-1]] * 5 + [want_no_boost], (rank, heads_fused)
        assert head_no_boost == want_no_boost, rank
        assert len(res) == N_EPOCHS and guard == 0
        for k, (okb, head) in enumerate(res):
            assert np.array_equal(np.frombuffer(okb, dtype=np.uint8), expect_ok), (rank, k)
            assert head == want_heads[k], (rank, k)
        assert lmd == want_lmd, rank
        assert head_again == want_heads[-1], rank
        for a, sig in agg_sample.items():
            assert sig == B.Sign(bench.committee_secret_sum(Wo, a), msgs[a]), (rank, a)
    assert all(r[2] == results[0][2] for r in results)
