"""N>1 host logic on CPU (world_size 2, gloo): validators sharded by rank, per-rank direct vote weights summed with
ONE all_reduce of int64[n_blocks], head computed on every rank from the reduced vector -- must equal the unsharded
result for any partition (SURVEY.md section 8e).  The GPU kernels are replaced by the numpy oracle behind the same
EpochProcessor plumbing (engine interface duck-typed), so what is tested is the sharding + collective, not the math."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenarios
from oracle import fast

N_VAL, N_BLK = 4096, 300


class _OracleEngine:
    """Duck-typed stand-in for engine.Engine: votes/head by the numpy oracle, BLS stages accept everything."""
    device = 0

    def __init__(self, tree, shard):
        self.parent, self.roots, self.leaf_viable = tree
        self.shard = shard

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        d_ok.fill_(1)

    def vote_weights_dev(self, d_votes):
        msg_block, has_msg, equiv, active, eff = self.shard
        w = np.zeros(N_BLK, dtype=np.uint64)
        m = (has_msg != 0) & (active != 0) & (equiv == 0)
        np.add.at(w, msg_block[m].astype(np.int64), eff[m])
        d_votes.copy_(torch.from_numpy(w.astype(np.int64)))

    def head_from_votes_dev(self, d_votes, d_head, justified_idx=0, boost_idx=-1, boost_score=0, d_weight=None):
        w = d_votes.numpy().astype(np.uint64).copy()
        if boost_idx >= 0:
            w[boost_idx] += np.uint64(boost_score)
        for b in range(N_BLK - 1, 0, -1):
            w[self.parent[b]] += w[b]
        d_head[0] = fast.ghost_head(self.parent, self.roots, fast.ghost_viable(self.parent, self.leaf_viable), w, justified_idx)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pos_evolution_b200.epoch import EpochProcessor
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    votes = scenarios.votes(N_VAL, N_BLK, 8)
    lo, hi = rank * N_VAL // world, (rank + 1) * N_VAL // world
    shard = tuple(v[lo:hi] for v in votes)
    ep = EpochProcessor(_OracleEngine((parent, roots, leaf_viable), shard), n_agg=4, n_sig=8, bits_stride=1, n_blocks=N_BLK,
                        process_group=dist.group.WORLD, device=torch.device("cpu"))
    ep.set_committees(np.arange(8, dtype=np.uint32), np.array([0, 2, 4, 6, 8], dtype=np.uint32))
    z = torch.zeros(1)
    ok, head = ep.process_epoch_dev(z, z, z, z, z, 0, N_BLK - 1, 12345)
    q.put((rank, int(head[0]), int(ok.sum())))
    dist.destroy_process_group()


def test_two_rank_sharding_equals_unsharded():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    msg_block, has_msg, equiv, active, eff = scenarios.votes(N_VAL, N_BLK, 8)
    w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, N_BLK - 1, 12345)
    expect = fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0)
    assert [r[1] for r in res] == [expect, expect]
    assert [r[2] for r in res] == [4, 4]


# ------------------------------------------------------------------------------------------ sharded epoch (strong scaling)
# ONE validator set, ONE epoch: rank g verifies only the aggregates of its slots, verdicts + aggregate signatures are
# all-gathered, every rank applies update_latest_messages for all accepted aggregates, votes are scattered by validator
# range and all-reduced.  The stand-in engine does the per-rank "GPU" work with numpy; what is tested is the slicing,
# the exchange and the order of operations of EpochProcessor's sharded mode against the unsharded sequential oracle.
S_VAL, S_AGG, S_CS = 1024, 8, 128


def _sharded_inputs():
    rng = np.random.default_rng(21)
    members = rng.permutation(S_VAL).astype(np.uint32)
    off = (np.arange(S_AGG + 1) * S_CS).astype(np.uint32)
    bits = rng.integers(0, 256, size=(S_AGG, S_CS // 8), dtype=np.uint8)
    verdict = np.array([1, 1, 0, 1, 1, 1, 0, 1], dtype=np.uint8)            # the two rejected aggregates sit on different ranks
    epochs = np.array([3, 3, 3, 4, 3, 3, 3, 3], dtype=np.int64)
    blocks = np.array([10, 20, 30, 40, 50, 60, 70, 80], dtype=np.int32)
    return members, off, bits, verdict, epochs, blocks


class _ShardEngine:
    """Stand-in for engine.Engine in sharded mode: verdicts come from a table keyed by the (global) message byte of each
    aggregate; the LMD table and the vote scatter are the numpy oracle over this rank's replica."""
    device = 0

    def __init__(self, tree, votes, verdict):
        self.parent, self.roots, self.leaf_viable = tree
        self.msg_block, self.has_msg, self.equiv, self.active, self.eff = [v.copy() for v in votes]
        self.msg_epoch = np.ones(S_VAL, dtype=np.uint64)
        self.verdict = verdict
        self.calls = []

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        assert d_target_epoch is None and d_block_idx is None, "a sharded epoch must not update the LMD table before the exchange"
        n = d_off.numel() - 1
        assert d_sigs.shape[0] == int(d_off[-1]) == d_members.numel() and d_bits.shape[0] == n == d_msgs.shape[0]
        for i in range(n):
            a = int(d_msgs[i, 0])                                            # global aggregate id travels in the message
            d_ok[i] = int(self.verdict[a])
            d_agg_sig.view(n, 96)[i] = a + 100                               # "aggregate signature" = recognisable bytes
        self.calls.append(("epoch", n))

    def latest_messages_update_dev(self, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_accept):
        members, off, bits = d_members.numpy().astype(np.uint32), d_off.numpy(), d_bits.numpy()
        assert len(off) - 1 == S_AGG, "every rank applies the LMD update for ALL aggregates of the epoch"
        for a in range(S_AGG):
            if not int(d_accept[a]):
                continue
            sel = [int(members[off[a] + j]) for j in range(off[a + 1] - off[a]) if (bits[a, j >> 3] >> (j & 7)) & 1]
            fast.lmd_update(self.msg_epoch, self.msg_block, self.has_msg, self.equiv, sel, int(d_target_epoch[a]), int(d_block_idx[a]))
        self.calls.append(("lmd", S_AGG))

    def vote_weights_range_dev(self, v0, v1, d_votes):
        w = np.zeros(N_BLK, dtype=np.uint64)
        m = (self.has_msg[v0:v1] != 0) & (self.active[v0:v1] != 0) & (self.equiv[v0:v1] == 0)
        np.add.at(w, self.msg_block[v0:v1][m].astype(np.int64), self.eff[v0:v1][m])
        d_votes.copy_(torch.from_numpy(w.astype(np.int64)))
        self.calls.append(("votes", v1 - v0))

    head_from_votes_dev = _OracleEngine.head_from_votes_dev


def _sharded_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pos_evolution_b200.epoch import EpochProcessor
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    votes = scenarios.votes(S_VAL, N_BLK, 8)
    members, off, bits, verdict, epochs, blocks = _sharded_inputs()
    eng = _ShardEngine((parent, roots, leaf_viable), votes, verdict)
    ep = EpochProcessor(eng, n_agg=S_AGG, n_sig=S_VAL, bits_stride=S_CS // 8, n_blocks=N_BLK, process_group=dist.group.WORLD,
                        device=torch.device("cpu"), shard=(rank, world), n_validators=S_VAL)
    ep.set_committees(members, off)
    assert (ep.a0, ep.a1) == (rank * S_AGG // world, (rank + 1) * S_AGG // world) and ep.n_sig_loc == S_VAL // world
    sigs = torch.zeros((S_VAL, 96), dtype=torch.uint8)
    msgs = torch.zeros((S_AGG, 32), dtype=torch.uint8)
    msgs[:, 0] = torch.arange(S_AGG, dtype=torch.uint8)
    ok, head = ep.process_epoch_dev(ep.local_signatures(sigs), torch.from_numpy(bits), msgs, torch.from_numpy(epochs), torch.from_numpy(blocks),
                                    0, N_BLK - 1, 12345)
    q.put((rank, int(head[0]), ok.tolist(), ep.d_agg_sig[0][:, 0].tolist(), eng.msg_epoch.tolist(), eng.msg_block.tolist(), eng.calls))
    dist.destroy_process_group()


def test_two_rank_sharded_epoch_equals_unsharded():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    # unsharded sequential oracle
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    msg_block, has_msg, equiv, active, eff = [v.copy() for v in scenarios.votes(S_VAL, N_BLK, 8)]
    members, off, bits, verdict, epochs, blocks = _sharded_inputs()
    msg_epoch = np.ones(S_VAL, dtype=np.uint64)
    for a in range(S_AGG):
        if verdict[a]:
            sel = [int(members[off[a] + j]) for j in range(S_CS) if (bits[a, j >> 3] >> (j & 7)) & 1]
            fast.lmd_update(msg_epoch, msg_block, has_msg, equiv, sel, int(epochs[a]), int(blocks[a]))
    w = fast.ghost_weights(parent, msg_block, has_msg, eff, active, equiv, N_BLK - 1, 12345)
    expect = fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0)
    for rank, head, ok, aggb, m_epoch, m_block, calls in res:
        assert head == expect
        assert ok == verdict.tolist()                                  # the all-gathered verdict vector, in aggregate order
        assert aggb == [a + 100 for a in range(S_AGG)]                 # the all-gathered aggregate signatures, in aggregate order
        assert m_epoch == msg_epoch.tolist() and m_block == msg_block.tolist()     # every replica of the LMD table == sequential rule
        assert calls == [("epoch", S_AGG // 2), ("lmd", S_AGG), ("votes", S_VAL // 2)]
