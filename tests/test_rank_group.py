"""tests/rank_group.py on CPU: the host-staged collectives of the shared_device layout against the plain gloo ones at world 2 and 3,
into contiguous tensors and into non-contiguous views of larger buffers; and `run`, which must fail fast and leave no rank behind
when one rank raises, dies without reporting or hangs."""
import multiprocessing
import os
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist

import rank_group

N = 7


def _inputs(rank):
    rng = np.random.default_rng(30 + rank)
    return (torch.from_numpy(rng.integers(0, 256, size=N, dtype=np.uint8)),
            torch.from_numpy(rng.integers(-2**62, 2**62, size=N, dtype=np.int64)))


def _collectives(world, x8, x64):
    """all_gather_into_tensor of uint8 and all_reduce of int64 (the product's two, the latter also with ReduceOp.MAX), each into a fresh
    contiguous tensor"""
    out = torch.zeros(world * N, dtype=torch.uint8)
    dist.all_gather_into_tensor(out, x8, group=dist.group.WORLD)
    red = x64.clone()
    dist.all_reduce(red, group=dist.group.WORLD)
    mx = x64.clone()
    dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=dist.group.WORLD)
    return [t.tolist() for t in (out, red, mx)]


def _into_views(world, x8, x64):
    """the same collectives into strided views of sentinel-filled buffers (which plain gloo refuses); -> the whole buffers"""
    buf8 = torch.full((world, 2 * N), 0xEE, dtype=torch.uint8)
    dist.all_gather_into_tensor(buf8[:, 1::2], x8, group=dist.group.WORLD)
    buf64 = torch.full((2 * N,), -5, dtype=torch.int64)
    buf64[::2] = x64
    dist.all_reduce(buf64[::2], group=dist.group.WORLD)
    return buf8.tolist(), buf64.tolist()


def _staging_worker(rank, world, port, q):
    rank_group.init_cpu(rank, world, port)
    x8, x64 = _inputs(rank)
    plain = _collectives(world, x8, x64)
    rank_group.stage_collectives()
    rank_group.stage_collectives()                    # idempotent: staged once, not twice
    assert dist.all_gather_into_tensor.staged.__name__ == "all_gather_into_tensor" and dist.all_reduce.staged.__name__ == "all_reduce"
    staged = _collectives(world, x8, x64)
    views = _into_views(world, x8, x64)
    q.put((rank, plain, staged, views))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_staged_collectives_equal_plain(world):
    res = rank_group.run(_staging_worker, world, timeout=300)
    assert [r[0] for r in res] == list(range(world))
    ins = [_inputs(r) for r in range(world)]
    gathered = torch.cat([x8 for x8, _ in ins])
    total = sum(x64 for _, x64 in ins)                # int64 wraps as the u64 vote sums do
    want = [gathered.tolist(), total.tolist(), torch.stack([x64 for _, x64 in ins]).max(0).values.tolist()]
    for rank, plain, staged, (buf8, buf64) in res:
        assert plain == want, rank
        assert staged == want, rank
        assert [row[1::2] for row in buf8] == gathered.view(world, N).tolist(), rank
        assert all(v == 0xEE for row in buf8 for v in row[0::2]), rank
        assert buf64[::2] == total.tolist() and buf64[1::2] == [-5] * N, rank


def _failing_worker(rank, world, port, q, how):
    if rank == 1:
        if how == "raise":
            raise ValueError("rank 1 gives up")
        if how == "exit":
            os._exit(7)                               # dies without a Python exception and without reporting
    if how == "hang" or rank != 1:
        time.sleep(600)
    q.put((rank,))


@pytest.mark.parametrize("how,timeout,error", [("raise", 60, "rank 1 gives up"), ("exit", 60, "exit code 7"), ("hang", 10, "ranks reported within")])
def test_run_fails_fast_and_leaves_no_rank_behind(how, timeout, error):
    t0 = time.monotonic()
    with pytest.raises((RuntimeError, TimeoutError)) as e:
        rank_group.run(_failing_worker, 3, args=(how,), timeout=timeout)
    assert error in str(e.value)
    assert time.monotonic() - t0 < 120                # the other ranks sleep for 600 s
    assert multiprocessing.active_children() == []


def _ok_worker(rank, world, port, q):
    q.put((rank, os.getpid()))


def test_run_returns_every_rank_in_order():
    res = rank_group.run(_ok_worker, 4, timeout=300)
    assert [r[0] for r in res] == [0, 1, 2, 3] and len({r[1] for r in res}) == 4
    assert multiprocessing.active_children() == []
