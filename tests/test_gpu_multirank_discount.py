"""Equivocation discounting in the sharded epoch pipeline, every rank a process with its own context.  Every rank runs the sharded
EpochProcessor with enable_slasher(..., discount=True) (pipelined, depth 3) on the six epochs of test_gpu_epoch_slasher.py: it marks the
equivocators of its own validator range, all-gathers its slice of the table padded to ceil(N / world) and merges the other ranks' slices
over their floor ranges.  Every rank's equivocating table and latest messages must be identical, and equal a single-process unsharded
run of the same epochs; so must the heads.

Two layouts (tests/rank_group.py): per_device, world 2 with one GPU per rank over NCCL (skipped below 2 GPUs); shared_device, the
ranks sharing one GPU over host-staged gloo, at world 2 and 4, and at world 4 on a registry of 67 validators (three in no committee),
where the padded slices and the floor ranges differ.  The shared layout runs the device path of the slice, the gather and the merge
before the next epoch's exchange, but not NCCL, NVLink or any multi-GPU timing."""
import numpy as np
import pytest

import rank_group

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _worker(rank, world, port, q, shared, n_val):
    import torch.distributed as dist
    import test_gpu_epoch_slasher as T
    from pos_evolution_b200.epoch import EpochProcessor
    dev = rank_group.init(rank, world, port, shared)
    members, off, tree, eff = T._world(n_val)
    eng = T._engine(tree, eff, dev.index)
    epochs = T._inputs(eng, members, off)
    ep = EpochProcessor(eng, T.N_AGG, T.N_AGG * T.CSIZE, 1, T.N_BLK, process_group=dist.group.WORLD, device=dev, depth=3,
                        shard=(rank, world), n_validators=n_val)
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


@pytest.mark.parametrize("layout,world,n_val", [("per_device", 2, 64), ("shared_device", 2, 64), ("shared_device", 4, 64), ("shared_device", 4, 67)])
def test_sharded_discount_equals_unsharded(layout, world, n_val):
    import test_gpu_epoch_discount as D
    if layout == "per_device" and torch.cuda.device_count() < world:
        pytest.skip("needs >= %d GPUs" % world)
    results = rank_group.run(_worker, world, args=(layout == "shared_device", n_val))
    whole, (equiv, e_, b_, h_) = D._six_epochs("pipelined", 3, True, n_val=n_val)
    assert len(equiv) == n_val and (equiv != 0).sum() == 12        # the four double voters of epoch 2 and eight surrounders of epoch 3
    for rank, heads, r_equiv, (r_e, r_b, r_h), guard in results:
        assert guard == 0, rank
        assert heads == [r[1] for r in whole], rank
        assert np.array_equal(r_equiv != 0, equiv != 0), rank
        assert np.array_equal(r_e, e_) and np.array_equal(r_b, b_) and np.array_equal(r_h, h_), rank
        assert np.array_equal(r_equiv, results[0][2]), rank
