"""The ranks of the multi-rank tests: one spawned process per rank, in one of two layouts.

  * "per_device": rank g on device g, collectives over NCCL -- the layout of a box with one GPU per rank;
  * "shared_device": every rank on device 0, collectives over gloo on 127.0.0.1 with the CUDA tensors staged through host memory.
    Each rank still owns its context, streams, events and kernels, so one GPU runs the sharded device path end to end; the staged
    collectives deliver the values NCCL would.  They say nothing about NCCL, NVLink or multi-GPU timing.

`init` joins a rank to the group; `run` spawns the ranks of one test and collects what each puts on its queue."""
import os
import queue
import socket
import time
import traceback

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

LAYOUTS = ("per_device", "shared_device")


def _staged(real, n_out):
    """`real` (a torch.distributed collective whose first n_out tensor arguments are written) run on host copies: the inputs are copied
    to host on the current stream (which waits for their producers, as an NCCL op enqueued on that stream would), the collective runs
    on flat contiguous host tensors, and its results are copied back into the caller's tensors (views of any shape included) on the
    current stream."""
    def collective(*tensors, **kw):
        host = [t.to("cpu", memory_format=torch.contiguous_format, copy=True).view(-1) for t in tensors]
        work = real(*host, **kw)
        if work is not None:                          # async_op=True: the copies back need the result
            work.wait()
        for t, h in zip(tensors[:n_out], host[:n_out]):
            t.copy_(h.view(t.shape))
        return work
    collective.staged = real
    return collective


def stage_collectives():
    """Replace torch.distributed.all_gather_into_tensor and all_reduce, in this process only, by their host-staged forms (the product
    looks both up on torch.distributed at call time).  Idempotent."""
    if not hasattr(dist.all_gather_into_tensor, "staged"):
        dist.all_gather_into_tensor = _staged(dist.all_gather_into_tensor, 1)
    if not hasattr(dist.all_reduce, "staged"):
        dist.all_reduce = _staged(dist.all_reduce, 1)


def _env(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))


def init(rank, world, port, shared):
    """Join rank `rank` of `world` to the default process group; returns the rank's device.  shared=False: device `rank` over NCCL.
    shared=True: device 0 over gloo, with the collectives staged through host memory (stage_collectives)."""
    _env(rank, world, port)
    if not shared:
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", device_id=dev)
        return dev
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")
    stage_collectives()
    return dev


def init_cpu(rank, world, port):
    """Join a CPU-only rank to a gloo group (the test of this module)."""
    _env(rank, world, port)
    dist.init_process_group("gloo")


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _entry(worker, rank, world, port, q, args):
    try:
        worker(rank, world, port, q, *args)
    except BaseException:
        q.put(("rank failed", rank, traceback.format_exc()))
        raise


def _stop(procs):
    for p in procs:
        if p.is_alive():
            p.terminate()
    for p in procs:
        p.join(timeout=30)
        if p.is_alive():
            p.kill()
            p.join()


def run(worker, world, args=(), timeout=900):
    """Spawn worker(rank, world, port, q, *args) for every rank and return the one item each rank puts on q, sorted by rank (items
    are tuples whose first element is the rank).  On a failing rank, a rank that ends without reporting, or no result within
    `timeout` seconds, every rank is terminated and joined before this raises; on success every rank must exit with code 0."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_entry, args=(worker, r, world, port, q, tuple(args))) for r in range(world)]
    results = []
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + timeout
        while len(results) < world:
            try:
                item = q.get(timeout=1.0)
            except queue.Empty:
                dead = [(r, p.exitcode) for r, p in enumerate(procs) if p.exitcode is not None and p.exitcode != 0]
                if dead:
                    raise RuntimeError("rank %d ended with exit code %s before reporting" % dead[0])
                if time.monotonic() > deadline:
                    raise TimeoutError("%d of %d ranks reported within %d s" % (len(results), world, timeout))
                continue
            if item[0] == "rank failed":
                raise RuntimeError("rank %d failed:\n%s" % item[1:])
            results.append(item)
        for r, p in enumerate(procs):
            p.join(timeout=max(1.0, deadline - time.monotonic()) + 60)
            assert p.exitcode == 0, "rank %d exited with %s" % (r, p.exitcode)
    finally:
        _stop(procs)
        q.close()
        q.join_thread()
    return sorted(results, key=lambda item: item[0])
