"""The vote form of the sharded epoch pipeline, every rank a process with its own context.  Every rank runs the sharded EpochProcessor
(pipelined, depth 3) on the split epochs of test_gpu_epoch_votes.py, whose ranks hold different numbers of votes: the verdicts, aggregate
signatures and aggregation bits of every vote, the heads and every rank's latest messages must equal a single-process unsharded run of
the same epochs.

Two layouts (tests/rank_group.py): per_device, world 2 with one GPU per rank over NCCL (skipped below 2 GPUs); shared_device, the
ranks sharing one GPU over host-staged gloo, at world 2, 3 and 6 (at 3 and 6 the ranks' vote counts differ from the padded width of the
all-gather), and at world 3 on a registry of 50 validators (two in no committee), whose validator ranges are uneven.  The shared layout
runs the device path of the grouping with per-rank segment offsets, the padded gather and the range scatter, but not NCCL, NVLink or
any multi-GPU timing."""
import numpy as np
import pytest

import rank_group

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _run(eng, dev, ep, T, members, off, vote_offs=None):
    out, keep = [], []
    for k in range(T.N_EPOCHS):
        E = T._epoch(eng, k, members, off)
        if vote_offs is not None:
            vote_offs.append(E["vote_off"])
        d = [torch.as_tensor(ep.local_signatures(E["sigs"]), device=dev), None] + [torch.as_tensor(E[x], device=dev) for x in ("msgs", "te", "bi")]
        dv = torch.as_tensor(E["vote"].view(np.int32), device=dev)
        keep.append((d, dv))
        t = ep.submit_dev(*d, last=k == T.N_EPOCHS - 1, votes=(dv, E["vote_off"]))
        for t in ([t] if t is not None else []) + (ep.drain() if k == T.N_EPOCHS - 1 else []):
            ok, hd = t.wait()
            out.append((ok.cpu().numpy().tolist(), hd, t.aggregate_signatures().cpu().numpy().tobytes(), t.aggregation_bits().cpu().numpy().tobytes()))
    torch.cuda.synchronize()
    return out, eng.latest_messages_read()


def _setup(dev, T, n_val, pg=None, shard=None):
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    pks, members, off, tree, eff = T._world(n_val)
    eng = Engine(dev.index)
    eng.registry_load(np.frombuffer(b"".join(pks), dtype=np.uint8), eff)
    eng.tree_load(*tree)
    eng.latest_messages_reset()
    ep = EpochProcessor(eng, T.N_C, len(members), 1, T.N_BLK, process_group=pg, device=dev, depth=3, shard=shard, n_validators=n_val,
                        max_votes=3 * T.N_C)
    ep.set_committees(members, off)
    return eng, ep, members, off


def _worker(rank, world, port, q, shared, n_val):
    import torch.distributed as dist
    import test_gpu_epoch_votes as T
    dev = rank_group.init(rank, world, port, shared)
    eng, ep, members, off = _setup(dev, T, n_val, dist.group.WORLD, (rank, world))
    out, lmd = _run(eng, dev, ep, T, members, off)
    q.put((rank, out, lmd, eng.guard_flags(), (ep.v0, ep.v1)))
    dist.barrier()
    dist.destroy_process_group()
    eng.close()


@pytest.mark.parametrize("layout,world,n_val", [("per_device", 2, 48), ("shared_device", 2, 48), ("shared_device", 3, 48), ("shared_device", 6, 48),
                                                ("shared_device", 3, 50)])
def test_sharded_vote_form_equals_unsharded(layout, world, n_val):
    import test_gpu_epoch_votes as T
    if layout == "per_device" and torch.cuda.device_count() < world:
        pytest.skip("needs >= %d GPUs" % world)
    results = rank_group.run(_worker, world, args=(layout == "shared_device", n_val))
    eng, ep, members, off = _setup(torch.device("cuda", 0), T, n_val)
    vote_offs = []
    want, (e_, b_, h_) = _run(eng, torch.device("cuda", 0), ep, T, members, off, vote_offs)
    eng.close()
    counts = [np.diff(vo[::T.N_C // world]) for vo in vote_offs]        # every rank's vote count, per epoch
    assert any(len(set(c.tolist())) > 1 for c in counts)               # some rank's block of the gather is padded
    assert [r[4] for r in results] == [(g * n_val // world, (g + 1) * n_val // world) for g in range(world)]
    for rank, out, (r_e, r_b, r_h), guard, _ in results:
        assert guard == 0, rank
        assert out == want, rank
        assert np.array_equal(r_h, h_) and np.array_equal(r_e[h_ == 1], e_[h_ == 1]) and np.array_equal(r_b[h_ == 1], b_[h_ == 1]), rank
