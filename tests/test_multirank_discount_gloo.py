"""Equivocation discounting in the sharded epoch pipeline, on CPU (world 2, gloo): where EpochProcessor puts the discount's calls.  A
stand-in engine (the one of test_multirank_slasher_gloo.py, plus the discount, slice and merge calls over a host copy of the equivocating
table) records every call; the processor runs the pipelined form at depth 3 and the synchronous form.  The registry has an odd number of
validators, so the ranks' ranges differ in length and the gathered slices are padded.  Checked:
  * each rank's discount follows its slasher update, with the update's kind vector and the whole epoch's members;
  * the rank's slice [v0, v1) is all-gathered, padded to ceil(N / world), and the other rank's row is merged over exactly its range;
  * the merge comes before the next epoch's exchange LMD update, so every replica of the table is identical at every epoch;
  * with discounting off, none of these calls appears."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import test_multirank_slasher_gloo as G

N_VAL = G.S_AGG * G.S_CS + 1                   # 257: members are the first 256 of a permutation of 257 validators


def _members():
    return np.random.default_rng(5).permutation(N_VAL)[:G.S_AGG * G.S_CS].astype(np.uint32)


class _DiscountEngine(G._SlasherEngine):
    n_validators = N_VAL

    def __init__(self):
        super().__init__()
        self.equiv = np.zeros(N_VAL, dtype=np.uint8)

    def latest_messages_update_dev(self, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_accept):
        self.calls.append(("lmd", d_accept.numpy().tobytes(), self.equiv.tobytes()))

    def slasher_discount_dev(self, d_members, d_kind, d_new, d_n_new):
        members, kind = d_members.numpy().astype(np.int64), d_kind.numpy()
        d_new.zero_()
        n = 0
        for i in np.nonzero(kind)[0]:
            if not self.equiv[members[i]]:
                self.equiv[members[i]] = 1
                d_new[i] = 1
                n += 1
        d_n_new[0] = n
        self.calls.append(("discount", members.tobytes(), kind.tobytes()))

    def equivocating_slice_dev(self, v_begin, v_end, d_out):
        d_out[:v_end - v_begin] = torch.from_numpy(self.equiv[v_begin:v_end].copy())
        self.calls.append(("slice", v_begin, v_end, d_out.numel()))

    def equivocating_merge_dev(self, v_begin, v_end, d_table):
        self.equiv[v_begin:v_end] |= d_table.numpy()[:v_end - v_begin]
        self.calls.append(("merge", v_begin, v_end, d_table.numpy().tobytes()))


def _worker(rank, world, port, q, mode, discount):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.current_stream = lambda *a, **k: G._Stream()         # no device in this process: stream order is call order
    torch.cuda.Event = G._Event
    from pos_evolution_b200.epoch import EpochProcessor
    eng = _DiscountEngine()
    ep = EpochProcessor(eng, n_agg=G.S_AGG, n_sig=G.S_AGG * G.S_CS, bits_stride=G.S_CS // 8, n_blocks=G.N_BLK, process_group=dist.group.WORLD,
                        device=torch.device("cpu"), depth=G.DEPTH, shard=(rank, world), n_validators=N_VAL)
    off = G._inputs(0)[1]
    ep.set_committees(_members(), off)
    ep.enable_slasher(64, current_epoch=G.CURS[0], discount=discount)
    found = []
    sigs = torch.zeros((G.S_AGG * G.S_CS, 96), dtype=torch.uint8)
    for k in range(len(G.CURS)):
        _, _, bits, _, src, tgt, msgs = G._inputs(k)
        args = (ep.local_signatures(sigs), torch.from_numpy(bits), torch.from_numpy(msgs), torch.from_numpy(tgt), torch.zeros(G.S_AGG, dtype=torch.int32))
        kw = dict(source_epoch=torch.from_numpy(src), current_epoch=G.CURS[k])
        if mode == "sync":
            ep.process_epoch_dev(*args, **kw)
            found.append(ep.discounted().tolist() if discount else None)
        else:
            t = ep.submit_dev(*args, last=(k == len(G.CURS) - 1), **kw)
            if t is not None:
                found.append(t.discounted().tolist() if discount else None)
    if mode != "sync":
        found += [t.discounted().tolist() if discount else None for t in ep.drain()]
    q.put((rank, (ep.v0, ep.v1), eng.calls, found, eng.equiv.tobytes()))
    dist.destroy_process_group()


def _run(mode, discount):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, mode, discount)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def _flagged(k, v0, v1):
    """the validators of [v0, v1) the stand-in slasher flags in epoch k: accepted aggregates whose span is not 1"""
    members = _members()
    _, off, bits, verdict, src, tgt, _ = G._inputs(k)
    out = set()
    for a in range(G.S_AGG):
        if verdict[a] and tgt[a] - src[a] != 1:
            out |= {int(members[off[a] + j]) for j in range(G.S_CS) if (bits[a, j >> 3] >> (j & 7)) & 1 and v0 <= members[off[a] + j] < v1}
    return out


def _check(res):
    width = -(-N_VAL // 2)
    ranges = [(g * N_VAL // 2, (g + 1) * N_VAL // 2) for g in range(2)]
    marked = set()
    lmd_tables = []
    for rank, (v0, v1), calls, found, equiv in res:
        assert (v0, v1) == ranges[rank]
        other = ranges[1 - rank]
        seq = [c for c in calls[1:] if c[0] in ("lmd", "slasher", "discount", "slice", "merge")]
        epochs, cur = [], None
        for c in seq:
            if c[0] == "lmd":
                cur = [c]
                epochs.append(cur)
            else:
                cur.append(c)
        assert len(epochs) == len(G.CURS)
        seen = set()
        tables = []
        for k, ev in enumerate(epochs):
            assert [c[0] for c in ev] == ["lmd", "slasher", "discount", "slice", "merge"], (k, [c[0] for c in ev])
            dc = ev[2]
            assert dc[1] == _members().astype(np.int64).tobytes()                   # the whole epoch's members ...
            kind = np.frombuffer(dc[2], dtype=np.uint8)
            assert set(_members()[kind != 0].tolist()) == _flagged(k, v0, v1)       # ... and the update's kind vector
            assert ev[3] == ("slice", v0, v1, width)                               # padded slice of the own range
            assert ev[4][1:3] == other                                             # the other rank's row, exactly its range
            got = np.frombuffer(ev[4][3], dtype=np.uint8)
            assert got.size == width and not got[other[1] - other[0]:].any()       # padding stays zero
            tables.append(ev[0][2])                                               # the table each exchange LMD update saw
            new = set(found[k])
            assert new == _flagged(k, v0, v1) - seen and all(v0 <= v < v1 for v in new), k
            seen |= new
        marked |= seen
        lmd_tables.append(tables)
        assert set(np.nonzero(np.frombuffer(equiv, dtype=np.uint8))[0].tolist()) >= seen
    # the merge of epoch k precedes the LMD update of epoch k+1 on both ranks, and both replicas are identical at every update
    assert lmd_tables[0] == lmd_tables[1]
    for k in range(1, len(G.CURS)):
        eq = np.frombuffer(lmd_tables[0][k], dtype=np.uint8)
        want = set().union(*(_flagged(j, 0, N_VAL) for j in range(k)))
        assert set(np.nonzero(eq)[0].tolist()) == want, k
    assert res[0][4] == res[1][4] and set(np.nonzero(np.frombuffer(res[0][4], dtype=np.uint8))[0].tolist()) == marked


def test_two_rank_sharded_discount_pipelined_depth3():
    _check(_run("pipelined", True))


def test_two_rank_sharded_discount_synchronous():
    _check(_run("sync", True))


def test_two_rank_sharded_without_discount_adds_no_call():
    for mode in ("pipelined", "sync"):
        for rank, _, calls, found, equiv in _run(mode, False):
            assert not {c[0] for c in calls} & {"discount", "slice", "merge"}
            assert found == [None] * len(G.CURS) and not any(equiv)
