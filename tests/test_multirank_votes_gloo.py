"""Vote form of the sharded epoch, host logic on CPU (world 2, gloo): every rank groups the whole epoch's indices and its own
committees' signatures, verifies the votes of its committees [vote_off[c0_g], vote_off[c1_g]) -- a different count per rank --, the
all-gather pads every rank's block to the largest count and unpacks it by vote, and every rank applies update_latest_messages over ALL
votes.  The result must equal the unsharded vote form and a sequential oracle.  The GPU kernels are replaced by a numpy stand-in behind
the same EpochProcessor plumbing (engine interface duck-typed, as test_multirank_gloo.py); its grouping is tests/votes_oracle.py, an
independent model of b2_votes_group_dev's layout."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenarios
import votes_oracle as VO
from oracle import fast

N_VAL, N_BLK, CS = 64, 50, 16
N_C = N_VAL // CS
NONE = 0xFFFFFFFF
VOTES_PER_COMMITTEE = [1, 3, 2, 1]               # rank 0: 4 votes, rank 1: 3 votes


def _inputs():
    rng = np.random.default_rng(7)
    members = rng.permutation(N_VAL).astype(np.uint32)
    off = (np.arange(N_C + 1) * CS).astype(np.uint32)
    vote_off = np.concatenate([[0], np.cumsum(VOTES_PER_COMMITTEE)]).astype(np.int64)
    n_votes = int(vote_off[-1])
    vote = np.full(N_VAL, NONE, dtype=np.uint32)
    for c in range(N_C):
        ids = vote_off[c] + rng.integers(0, VOTES_PER_COMMITTEE[c], size=CS)
        vote[off[c]:off[c + 1]] = np.where(rng.random(CS) < 0.2, NONE, ids)
    sigs = np.zeros((N_VAL, 96), dtype=np.uint8)
    sigs[:, 0] = members % 251 + 1                                       # a signature names its signer
    verdict = np.ones(n_votes, dtype=np.uint8)
    verdict[[2, 5]] = 0                                                  # one rejected vote on each rank
    epochs = np.full(n_votes, 3, dtype=np.int64)
    epochs[4] = 4
    blocks = (np.arange(n_votes) * 7 + 3).astype(np.int32)
    return members, off, vote, vote_off, sigs, verdict, epochs, blocks


class _VoteEngine:
    """Stand-in for engine.Engine: grouping in numpy, verdicts from a table keyed by the vote id carried in each message, the
    'aggregate signature' = (vote id, sum of its attesters' signer bytes), the LMD table and the vote scatter by the numpy oracle."""
    device = 0

    def __init__(self, tree, verdict):
        self.parent, self.roots, self.leaf_viable = tree
        self.msg_epoch, self.msg_block = np.zeros(N_VAL, dtype=np.uint64), np.zeros(N_VAL, dtype=np.uint32)
        self.has_msg, self.equiv = np.zeros(N_VAL, dtype=np.uint8), np.zeros(N_VAL, dtype=np.uint8)
        self.eff = np.full(N_VAL, 32, dtype=np.uint64)
        self.verdict = verdict
        self.calls = []

    def votes_group_dev(self, d_vote, d_vote_off, d_members, d_off, d_sigs, c_begin, c_end, d_sigs_out, d_members_out, d_pos_out, d_seg_off,
                        d_bits_out, d_agg_bits_out, d_seg_off_loc=None):
        vote, vote_off = d_vote.numpy().view(np.uint32), d_vote_off.numpy().astype(np.int64)
        members, off = d_members.numpy().view(np.uint32), d_off.numpy().astype(np.int64)
        n_votes = int(vote_off[-1])
        assert d_seg_off.numel() == n_votes + 1 and d_bits_out.shape[0] == n_votes
        g = VO.group_outputs(members, off, vote, vote_off, d_sigs.numpy(), d_bits_out.shape[1], c_begin, c_end)
        d_members_out.copy_(torch.from_numpy(g.members_out.view(np.int32)))
        d_pos_out.copy_(torch.from_numpy(g.pos_out.astype(np.int32)))
        d_seg_off.copy_(torch.from_numpy(g.seg_off.astype(np.int32)))
        d_bits_out.copy_(torch.from_numpy(g.bits))
        d_agg_bits_out.copy_(torch.from_numpy(g.agg_bits))
        d_sigs_out.copy_(torch.from_numpy(g.sigs_out))
        if d_seg_off_loc is not None:
            d_seg_off_loc[:g.seg_off_loc.shape[0]] = torch.from_numpy(g.seg_off_loc.astype(np.int32))
        self.calls.append(("group", c_begin, c_end))

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        n = d_off.numel() - 1
        off = d_off.numpy().astype(np.int64)
        assert d_sigs.shape[0] == off[-1] == d_members.numel() and d_bits.shape[0] == n == d_msgs.shape[0] and off[0] == 0
        sig = d_agg_sig.view(n, 96)
        for i in range(n):
            v = int(d_msgs[i, 0])
            seg = d_sigs[off[i]:off[i + 1], 0].numpy()
            d_ok[i] = int(self.verdict[v])
            sig[i] = 0
            sig[i, 0], sig[i, 1] = v + 100, int(seg[seg != 0xC0].astype(np.int64).sum() % 256)
        if d_target_epoch is not None:
            self.latest_messages_update_dev(d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_ok)
        self.calls.append(("epoch", n))

    def votes_empty_dev(self, d_bits, d_agg_sig, d_agg_status=None):
        n = d_bits.shape[0]
        empty = (d_bits[:, 0] & 1) == 0
        d_agg_sig.view(n, 96)[empty] = 0

    def latest_messages_update_dev(self, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_accept):
        members, off, bits = d_members.numpy().view(np.uint32), d_off.numpy(), d_bits.numpy()
        for a in range(len(off) - 1):
            if int(d_accept[a]):
                sel = [int(members[off[a] + j]) for j in range(off[a + 1] - off[a]) if (bits[a, j >> 3] >> (j & 7)) & 1]
                fast.lmd_update(self.msg_epoch, self.msg_block, self.has_msg, self.equiv, sel, int(d_target_epoch[a]), int(d_block_idx[a]))
        self.calls.append(("lmd", len(off) - 1))

    def vote_weights_range_dev(self, v0, v1, d_votes):
        w = np.zeros(N_BLK, dtype=np.uint64)
        m = (self.has_msg[v0:v1] != 0) & (self.equiv[v0:v1] == 0)
        np.add.at(w, self.msg_block[v0:v1][m].astype(np.int64), self.eff[v0:v1][m])
        d_votes.copy_(torch.from_numpy(w.astype(np.int64)))

    def vote_weights_dev(self, d_votes):
        self.vote_weights_range_dev(0, N_VAL, d_votes)

    def head_from_votes_dev(self, d_votes, d_head, justified_idx=0, boost_idx=-1, boost_score=0, d_weight=None):
        w = d_votes.numpy().astype(np.uint64).copy()
        for b in range(N_BLK - 1, 0, -1):
            w[self.parent[b]] += w[b]
        d_head[0] = fast.ghost_head(self.parent, self.roots, fast.ghost_viable(self.parent, self.leaf_viable), w, justified_idx)


def _run(rank, world, pg):
    from pos_evolution_b200.epoch import EpochProcessor
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    members, off, vote, vote_off, sigs, verdict, epochs, blocks = _inputs()
    n_votes = int(vote_off[-1])
    eng = _VoteEngine((parent, roots, leaf_viable), verdict)
    shard = (rank, world) if world > 1 else None
    ep = EpochProcessor(eng, n_agg=N_C, n_sig=N_VAL, bits_stride=CS // 8, n_blocks=N_BLK, process_group=pg, device=torch.device("cpu"),
                        shard=shard, n_validators=N_VAL, max_votes=8)
    ep.set_committees(members, off)
    msgs = torch.zeros((n_votes, 32), dtype=torch.uint8)
    msgs[:, 0] = torch.arange(n_votes, dtype=torch.uint8)
    ok, head = ep.process_epoch_dev(ep.local_signatures(torch.from_numpy(sigs)), None, msgs, torch.from_numpy(epochs), torch.from_numpy(blocks),
                                    votes=(torch.from_numpy(vote.view(np.int32)), vote_off))
    s = ep.slots[0]
    return (int(head[0]), ok.tolist(), s.agg_sig[:n_votes, :2].tolist(), s.v_aggbits[:n_votes].tolist(), eng.msg_epoch.tolist(), eng.msg_block.tolist(),
            eng.has_msg.tolist(), eng.calls, s.layout.ranges, s.layout.pad)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q.put((rank, _run(rank, world, dist.group.WORLD)))
    dist.destroy_process_group()


def _oracle():
    parent, slot, roots, leaf_viable = scenarios.fork_tree(N_BLK, 8)
    members, off, vote, vote_off, sigs, verdict, epochs, blocks = _inputs()
    n_votes = int(vote_off[-1])
    e, b, h, q = np.zeros(N_VAL, np.uint64), np.zeros(N_VAL, np.uint32), np.zeros(N_VAL, np.uint8), np.zeros(N_VAL, np.uint8)
    aggs = []
    for c in range(N_C):
        for v in range(int(vote_off[c]), int(vote_off[c + 1])):
            sel = [int(members[off[c] + j]) for j in range(CS) if vote[off[c] + j] == v]
            aggs.append([v + 100, sum(x % 251 + 1 for x in sel) % 256] if sel else [0, 0])
            if verdict[v]:
                fast.lmd_update(e, b, h, q, sel, int(epochs[v]), int(blocks[v]))
    w = fast.ghost_weights(parent, b, h, np.full(N_VAL, 32, dtype=np.uint64), np.ones(N_VAL, np.uint8), q, -1, 0)
    head = fast.ghost_head(parent, roots, fast.ghost_viable(parent, leaf_viable), w, 0)
    return head, verdict.tolist(), aggs, e.tolist(), b.tolist(), h.tolist(), n_votes


def test_two_rank_vote_form_equals_unsharded():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    single = _run(0, 1, None)
    head, verdict, aggs, e, b, h, n_votes = _oracle()
    assert single[:3] == (head, verdict, aggs) and single[4:7] == (e, b, h)
    members, off, vote, vote_off, *_ = _inputs()
    for rank in (0, 1):
        r = res[rank]
        assert r[0] == head and r[1] == verdict and r[2] == aggs             # the unpacked all-gather, in vote order
        assert r[3] == single[3]                                            # aggregation_bits of every vote, grouped on every rank
        assert r[4:7] == (e, b, h)                                          # every replica of the LMD table == sequential rule
        assert r[8] == [(0, 4), (4, 3)] and r[9] == 4                       # per-rank vote ranges, padded to the larger count
        c0, c1 = rank * N_C // 2, (rank + 1) * N_C // 2
        n_loc = int(vote_off[c1] - vote_off[c0])
        assert r[7] == [("group", c0, c1), ("epoch", n_loc), ("lmd", n_votes)]
