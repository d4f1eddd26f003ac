"""The vote form of the sharded epoch pipeline on real GPUs (needs >= 2; run with `python -m pytest tests/test_gpu_multirank_votes.py -m gpu`
on a machine with two or more H100s).  Every rank runs the sharded EpochProcessor over NCCL (pipelined, depth 3) on the split epochs of
test_gpu_epoch_votes.py, whose ranks hold different numbers of votes: the verdicts, aggregate signatures and aggregation bits of every
vote, the heads and every rank's latest messages must equal a single-process unsharded run of the same epochs."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _run(eng, dev, ep, T, members, off):
    out, keep = [], []
    for k in range(T.N_EPOCHS):
        E = T._epoch(eng, k, members, off)
        d = [torch.as_tensor(ep.local_signatures(E["sigs"]), device=dev), None] + [torch.as_tensor(E[x], device=dev) for x in ("msgs", "te", "bi")]
        dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
        keep.append((d, dv))
        t = ep.submit_dev(*d, last=k == T.N_EPOCHS - 1, votes=(dv, E["vote_off"]))
        for t in ([t] if t is not None else []) + (ep.drain() if k == T.N_EPOCHS - 1 else []):
            ok, hd = t.wait()
            out.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().tobytes(), t.aggregation_bits().cpu().numpy().tobytes()))
    torch.cuda.synchronize()
    return out, eng.latest_messages_read()


def _setup(rank, T, pg=None, shard=None):
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    dev = torch.device("cuda", rank)
    eng = Engine(rank)
    pks = T.scenarios.pubkeys(T.N_VAL)
    rng = np.random.default_rng(5)
    members = rng.permutation(T.N_VAL).astype(np.uint32)
    off = (np.arange(T.N_C + 1) * T.CSIZE).astype(np.uint32)
    eff = rng.integers(16, 33, size=T.N_VAL).astype(np.uint64) * np.uint64(10**9)
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(*T.scenarios.fork_tree(T.N_BLK, 5))
    eng.latest_messages_reset()
    ep = EpochProcessor(eng, T.N_C, T.N_VAL, 1, T.N_BLK, process_group=pg, device=dev, depth=3, shard=shard, n_validators=T.N_VAL,
                        max_votes=3 * T.N_C)
    ep.set_committees(members, off)
    return eng, dev, ep, members, off


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    import test_gpu_epoch_votes as T
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    eng, dev, ep, members, off = _setup(rank, T, dist.group.WORLD, (rank, world))
    out, lmd = _run(eng, dev, ep, T, members, off)
    q.put((rank, out, lmd, eng.guard_flags()))
    dist.barrier()
    dist.destroy_process_group()
    eng.close()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_vote_form_on_two_gpus_equals_unsharded():
    import torch.multiprocessing as mp
    import test_gpu_epoch_votes as T
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=900) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    eng, dev, ep, members, off = _setup(0, T)
    want, (e_, b_, h_) = _run(eng, dev, ep, T, members, off)
    eng.close()
    for rank, out, (r_e, r_b, r_h), guard in results:
        assert guard == 0, rank
        assert out == want, rank
        assert np.array_equal(r_h, h_) and np.array_equal(r_e[h_ == 1], e_[h_ == 1]) and np.array_equal(r_b[h_ == 1], b_[h_ == 1]), rank
