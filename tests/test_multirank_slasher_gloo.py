"""The slasher in the sharded epoch pipeline, on CPU (world 2, gloo): where EpochProcessor puts the slasher's calls.  A duck-typed
stand-in engine records every call; the processor runs the pipelined form at depth 3 (torch's stream and event calls are stubbed, as
there is no device) and the synchronous form.  What is checked is the plumbing, not the detection:
  * each rank initialises the history of its vote-scatter range [v0, v1) only;
  * per epoch, the update comes after the verdict exchange and the fork choice, with the all-gathered verdict bytes as accept and the
    whole epoch's members, offsets, bits, messages, source and target epochs;
  * the window moves (slasher_advance_dev) right before the update, and only when the epoch moved;
  * updates arrive in epoch order through the pipeline, and every rank's report covers its own range: together they are the
    unsharded report."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

N_BLK, S_VAL, S_AGG, S_CS, DEPTH = 50, 256, 8, 32, 3
# (current epoch, source offset) per epoch: the window stays put between epochs 1 and 2
CURS = [10, 11, 11, 12, 14, 15]


def _inputs(k):
    rng = np.random.default_rng(21)
    members = rng.permutation(S_VAL).astype(np.uint32)
    off = (np.arange(S_AGG + 1) * S_CS).astype(np.uint32)
    erng = np.random.default_rng(100 + k)
    bits = erng.integers(0, 256, size=(S_AGG, S_CS // 8), dtype=np.uint8)
    verdict = np.ones(S_AGG, dtype=np.uint8)
    verdict[(k + 2) % S_AGG] = 0
    verdict[(k + 5) % S_AGG] = 0                                          # one rejected aggregate on each rank
    cur = CURS[k]
    tgt = np.full(S_AGG, cur, dtype=np.int64)
    src = np.full(S_AGG, cur - 1, dtype=np.int64)
    src[k % S_AGG] = cur - 3                                              # the stand-in flags aggregates whose span is not 1
    msgs = np.zeros((S_AGG, 32), dtype=np.uint8)
    msgs[:, 0] = np.arange(S_AGG)
    msgs[:, 1] = k
    return members, off, bits, verdict, src, tgt, msgs


class _Stream:
    cuda_stream = 0

    def wait_event(self, ev):
        pass

    def synchronize(self):
        pass


class _Event:
    def record(self, stream=None):
        pass

    def synchronize(self):
        pass


class _SlasherEngine:
    """Stand-in for engine.Engine in sharded mode: verdicts from a per-epoch table keyed by the message bytes; every call recorded"""
    device = 0
    n_validators = S_VAL

    def __init__(self):
        self.calls = []
        self.pending = {}

    def epoch_set_pairing_form(self, team):
        pass

    def epoch_start_dev(self, slot, d_sigs, d_members, d_off, d_bits, d_msgs, d_agg_status):
        self.pending[slot] = d_msgs.clone()

    def epoch_tail_dev(self, slot, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        assert d_target_epoch is None and d_block_idx is None
        msgs = self.pending[slot]
        n = d_off.numel() - 1
        for i in range(n):
            a, k = int(msgs[i, 0]), int(msgs[i, 1])
            d_ok[i] = int(_inputs(k)[3][a])
            d_agg_sig.view(n, 96)[i] = a + 100

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        self.epoch_start_dev(0, d_sigs, d_members, d_off, d_bits, d_msgs, d_agg_status)
        self.epoch_tail_dev(0, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok)

    def epoch_wait_dev(self, slot):
        self.calls.append(("wait", slot))

    def latest_messages_update_dev(self, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_accept):
        self.calls.append(("lmd", d_accept.numpy().tobytes()))

    def vote_weights_range_dev(self, v0, v1, d_votes):
        d_votes.zero_()
        self.calls.append(("votes", v0, v1))

    def head_from_votes_dev(self, d_votes, d_head, justified_idx=0, boost_idx=-1, boost_score=0, d_weight=None):
        d_head[0] = 7
        self.calls.append(("head",))

    def slasher_init(self, n_validators, history_epochs, max_attestations_per_target, current_epoch=0, v_begin=0, v_end=None):
        self.range = (v_begin, v_end)
        self.calls.append(("init", n_validators, history_epochs, max_attestations_per_target, current_epoch, v_begin, v_end))

    def slasher_advance_dev(self, current_epoch):
        self.calls.append(("advance", current_epoch))

    def slasher_update_dev(self, d_members, d_off, d_bits, d_source_epoch, d_target_epoch, d_roots, d_accept, d_status, d_kind, d_conflict,
                           d_n_flagged):
        members, off, bits = d_members.numpy().astype(np.int64), d_off.numpy().astype(np.int64), d_bits.numpy()
        src, tgt, acc = d_source_epoch.numpy(), d_target_epoch.numpy(), d_accept.numpy()
        v0, v1 = self.range
        d_kind.zero_()
        d_conflict.fill_(-1)
        n = 0
        for a in range(len(off) - 1):
            d_status[a] = 0 if acc[a] else 1
            if not acc[a] or tgt[a] - src[a] == 1:
                continue
            for j in range(off[a + 1] - off[a]):
                v = members[off[a] + j]
                if (bits[a, j >> 3] >> (j & 7)) & 1 and v0 <= v < v1:
                    d_kind[off[a] + j] = 2
                    d_conflict[off[a] + j, 0] = int(tgt[a]) - 1
                    n += 1
        d_n_flagged[0] = n
        self.calls.append(("slasher", d_members.numpy().tobytes(), d_off.numpy().tobytes(), bits.tobytes(), d_roots.numpy().tobytes(),
                           src.tobytes(), tgt.tobytes(), acc.tobytes()))


def _worker(rank, world, port, q, mode):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.current_stream = lambda *a, **k: _Stream()         # no device in this process: stream order is call order
    torch.cuda.Event = _Event
    from pos_evolution_b200.epoch import EpochProcessor
    eng = _SlasherEngine()
    ep = EpochProcessor(eng, n_agg=S_AGG, n_sig=S_VAL, bits_stride=S_CS // 8, n_blocks=N_BLK, process_group=dist.group.WORLD,
                        device=torch.device("cpu"), depth=DEPTH, shard=(rank, world), n_validators=S_VAL)
    members, off = _inputs(0)[:2]
    ep.set_committees(members, off)
    ep.enable_slasher(64, current_epoch=CURS[0])
    reports = []
    tickets = []
    sigs = torch.zeros((S_VAL, 96), dtype=torch.uint8)
    for k in range(len(CURS)):
        _, _, bits, _, src, tgt, msgs = _inputs(k)
        args = (ep.local_signatures(sigs), torch.from_numpy(bits), torch.from_numpy(msgs), torch.from_numpy(tgt), torch.zeros(S_AGG, dtype=torch.int32))
        kw = dict(source_epoch=torch.from_numpy(src), current_epoch=CURS[k])
        if mode == "sync":
            ep.process_epoch_dev(*args, **kw)
            r = ep.slashings()
            reports.append((r.status.tolist(), r.aggregate.tolist(), r.position.tolist(), r.validator.tolist(), r.kind.tolist(),
                            r.surrounded_target.tolist()))
        else:
            t = ep.submit_dev(*args, last=(k == len(CURS) - 1), **kw)
            if t is not None:
                tickets.append(t)
                r = t.slashings()
                reports.append((r.status.tolist(), r.aggregate.tolist(), r.position.tolist(), r.validator.tolist(), r.kind.tolist(),
                                r.surrounded_target.tolist()))
    if mode != "sync":
        for t in ep.drain():
            r = t.slashings()
            reports.append((r.status.tolist(), r.aggregate.tolist(), r.position.tolist(), r.validator.tolist(), r.kind.tolist(),
                            r.surrounded_target.tolist()))
    q.put((rank, (ep.v0, ep.v1), eng.calls, reports))
    dist.destroy_process_group()


def _run(mode):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, mode)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def _check(res):
    union = [set() for _ in CURS]
    for rank, (v0, v1), calls, reports in res:
        assert (v0, v1) == (rank * S_VAL // 2, (rank + 1) * S_VAL // 2)
        assert calls[0] == ("init", S_VAL, 64, 2 * S_AGG, CURS[0], v0, v1)
        # split the call log into epochs at each "wait" that starts a fork-choice sequence
        seq = [c for c in calls[1:] if c[0] in ("lmd", "votes", "head", "advance", "slasher")]
        epochs, cur = [], None
        for c in seq:
            if c[0] == "lmd":
                cur = [c]
                epochs.append(cur)
            else:
                cur.append(c)
        assert len(epochs) == len(CURS)
        last = CURS[0]
        for k, ev in enumerate(epochs):
            members, off, bits, verdict, src, tgt, msgs = _inputs(k)
            moved = CURS[k] != last
            names = [c[0] for c in ev]
            assert names == ["lmd", "votes", "head"] + (["advance"] if moved else []) + ["slasher"], (k, names)
            if moved:
                assert ev[3] == ("advance", CURS[k])
            last = CURS[k]
            assert ev[0][1] == verdict.tobytes()                            # the LMD update used the gathered verdicts ...
            sl = ev[-1]
            assert sl[1] == members.astype(np.int32).tobytes() and sl[2] == off.astype(np.int32).tobytes()   # ... and so does the slasher,
            assert sl[3] == bits.tobytes() and sl[4] == msgs.tobytes()      # over the whole epoch, in epoch order
            assert sl[5] == src.tobytes() and sl[6] == tgt.tobytes() and sl[7] == verdict.tobytes()
            status, agg, pos, val, kind, surrounded = reports[k]
            assert status == [0 if x else 1 for x in verdict]
            assert all(v0 <= v < v1 for v in val) and set(kind) <= {2}
            assert all(int(members[off[a] + p]) == v for a, p, v in zip(agg, pos, val))
            assert all(t == CURS[k] - 1 for t in surrounded)
            assert not union[k] & set(val)
            union[k] |= set(val)
    for k in range(len(CURS)):                                              # the ranks' reports together: the unsharded one
        members, off, bits, verdict, src, tgt, msgs = _inputs(k)
        want = set()
        for a in range(S_AGG):
            if verdict[a] and tgt[a] - src[a] != 1:
                want |= {int(members[off[a] + j]) for j in range(S_CS) if (bits[a, j >> 3] >> (j & 7)) & 1}
        assert union[k] == want, k


def test_two_rank_sharded_slasher_pipelined_depth3():
    _check(_run("pipelined"))


def test_two_rank_sharded_slasher_synchronous():
    _check(_run("sync"))
