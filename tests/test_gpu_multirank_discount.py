"""Equivocation discounting in the sharded epoch pipeline on real GPUs (needs >= 2; run with
`python -m pytest tests/test_gpu_multirank_discount.py -m gpu` on a machine with two or more H100s).  Every rank runs the sharded
EpochProcessor over NCCL with enable_slasher(..., discount=True) (pipelined, depth 3) on the six epochs of test_gpu_epoch_slasher.py:
it marks the equivocators of its own validator range and merges the other ranks' slices.  Every rank's equivocating table and latest
messages must be identical, and equal a single-process unsharded run of the same epochs; so must the heads."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    import test_gpu_epoch_slasher as T
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    members, off, (parent, slot, roots, leaf_viable), eff = T._world()
    eng = Engine(rank)
    eng.registry_load(eng.sk_to_pk([T.scenarios.secret_key(v) for v in range(T.N_VAL)]), eff)
    eng.tree_load(parent, slot, roots, leaf_viable)
    eng.latest_messages_reset()
    epochs = T._inputs(eng, members, off)
    ep = EpochProcessor(eng, T.N_AGG, T.N_AGG * T.CSIZE, 1, T.N_BLK, process_group=dist.group.WORLD, device=dev, depth=3,
                        shard=(rank, world), n_validators=T.N_VAL)
    ep.set_committees(members, off)
    ep.enable_slasher(16, current_epoch=T.CUR0, discount=True)
    heads, keep = [], []
    for k, e in enumerate(epochs):
        d = [torch.as_tensor(ep.local_signatures(e["sigs"]), device=dev)] + [torch.as_tensor(e[x], device=dev) for x in ("bits", "msgs", "tgt", "blk")]
        src = torch.as_tensor(e["src"], device=dev)
        keep.append((d, src))
        t = ep.submit_dev(*d, last=(k == len(epochs) - 1), source_epoch=src, current_epoch=T.CUR0 + k)
        if t is not None:
            heads.append(t.wait()[1])
    heads += [t.wait()[1] for t in ep.drain()]
    torch.cuda.synchronize()
    q.put((rank, heads, ep.equivocating(), eng.latest_messages_read(), eng.guard_flags()))
    dist.barrier()
    dist.destroy_process_group()
    eng.close()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_discount_on_two_gpus_equals_unsharded():
    import torch.multiprocessing as mp
    import test_gpu_epoch_discount as D
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
    whole, (equiv, e_, b_, h_) = D._six_epochs("pipelined", 3, True)
    for rank, heads, r_equiv, (r_e, r_b, r_h), guard in results:
        assert guard == 0, rank
        assert heads == [r[1] for r in whole], rank
        assert np.array_equal(r_equiv != 0, equiv != 0), rank
        assert np.array_equal(r_e, e_) and np.array_equal(r_b, b_) and np.array_equal(r_h, h_), rank
    assert np.array_equal(results[0][2], results[1][2])
