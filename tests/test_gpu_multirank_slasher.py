"""The slasher in the sharded epoch pipeline, every rank a process with its own context.  Every rank runs the sharded EpochProcessor
with enable_slasher on the six epochs of test_gpu_epoch_slasher.py, so it holds the history of its validator range only; the union of
the ranks' flagged member slots must equal a single-process unsharded run of the same epochs in the same form, the ranks' slots must
lie in their ranges and every rank must report the same per-aggregate statuses.

Two layouts (tests/rank_group.py):
  * per_device: world 2, one GPU per rank over NCCL (skipped below 2 GPUs), pipelined (submit_dev, depth 3);
  * shared_device: the ranks share one GPU over host-staged gloo: pipelined at world 2 and 4, and the synchronous process_epoch_dev and
    process_epoch_host (sharded) at world 2.
The shared layout runs every device call of the sharded path -- the tail without the LMD update, the exchange's LMD update on the
fork-choice stream, the range scatter and the range slasher fed the gathered verdicts -- but not NCCL, NVLink or any multi-GPU timing."""
import numpy as np
import pytest

import rank_group

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _report(sl):
    rows = zip(sl.aggregate.tolist(), sl.position.tolist(), sl.validator.tolist(), sl.kind.tolist(), sl.surrounded_target.tolist(),
               sl.surrounding_target.tolist())
    return sl.status.tolist(), sorted(rows)


def _worker(rank, world, port, q, shared, mode):
    import torch.distributed as dist
    import test_gpu_epoch_slasher as T
    from pos_evolution_b200.epoch import EpochProcessor
    dev = rank_group.init(rank, world, port, shared)
    members, off, tree, eff = T._world()
    eng = T._engine(tree, eff, dev.index)
    epochs = T._inputs(eng, members, off)
    ep = EpochProcessor(eng, T.N_AGG, T.N_AGG * T.CSIZE, 1, T.N_BLK, process_group=dist.group.WORLD, device=dev, depth=3,
                        shard=(rank, world), n_validators=T.N_VAL)
    ep.set_committees(members, off)
    ep.enable_slasher(16, current_epoch=T.CUR0)
    out, keep = [], []
    for k, e in enumerate(epochs):
        d = [torch.as_tensor(ep.local_signatures(e["sigs"]), device=dev)] + [torch.as_tensor(e[x], device=dev) for x in ("bits", "msgs", "tgt", "blk")]
        src = torch.as_tensor(e["src"], device=dev)
        keep.append((d, src))
        if mode == "sync":
            ep.process_epoch_dev(*d, source_epoch=src, current_epoch=T.CUR0 + k)
            out.append(_report(ep.slashings()))
        elif mode == "sync_host":
            h, hs = [x.cpu().pin_memory() for x in d], src.cpu().pin_memory()
            keep.append((h, hs))
            ep.process_epoch_host(*h, source_epoch=hs, current_epoch=T.CUR0 + k)
            out.append(_report(ep.slashings()))
        else:
            t = ep.submit_dev(*d, last=(k == len(epochs) - 1), source_epoch=src, current_epoch=T.CUR0 + k)
            if t is not None:
                out.append(_report(t.slashings()))
    out += [_report(t.slashings()) for t in ep.drain()]
    q.put((rank, ep.sl_range, out, eng.guard_flags()))
    dist.barrier()
    dist.destroy_process_group()
    eng.close()


@pytest.mark.parametrize("layout,world,mode", [("per_device", 2, "pipelined"), ("shared_device", 2, "pipelined"), ("shared_device", 4, "pipelined"),
                                               ("shared_device", 2, "sync"), ("shared_device", 2, "sync_host")])
def test_sharded_slasher_equals_unsharded(layout, world, mode):
    import test_gpu_epoch_slasher as T
    if layout == "per_device" and torch.cuda.device_count() < world:
        pytest.skip("needs >= %d GPUs" % world)
    results = rank_group.run(_worker, world, args=(layout == "shared_device", mode))
    whole = [_report(r[3]) for r in T._run(mode, 3, 16, True)]
    assert [r[1] for r in results] == [(g * T.N_VAL // world, (g + 1) * T.N_VAL // world) for g in range(world)]
    for k in range(T.N_EPOCHS):
        union = []
        for rank, (v0, v1), out, guard in results:
            status, rows = out[k]
            assert guard == 0 and status == whole[k][0], (rank, k)
            assert all(v0 <= row[2] < v1 for row in rows), (rank, k)
            union += rows
        assert sorted(union) == whole[k][1], k
        assert len(union) == T.EXPECTED_FLAGGED.get(k, 0)
    assert np.array_equal([len(w[1]) for w in whole], [T.EXPECTED_FLAGGED.get(k, 0) for k in range(T.N_EPOCHS)])
