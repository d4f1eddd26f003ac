"""Throughput of bls.AggregateVerify on device-resident inputs (b2_aggregate_verify_dev), beside FastAggregateVerify
(b2_fast_aggregate_verify_dev) on as many aggregates.

    python tools/aggregate_verify_bench.py [--sets 2048] [--sizes 1,16,128] [--warmup 3] [--iters 10]

For each set size: 2 048 sets of that many (registry key, 32-byte message) pairs, signed on the GPU (bls.Sign per pair,
bls.Aggregate per set), every verdict checked to be 1; then CUDA-event timing of `iters` calls after `warmup` calls.  Reports
sets/s, pairs/s and the time per Miller loop (call time / (pairs + sets): everything of the call, the per-set final
exponentiations included, spread over its Miller loops); FastAggregateVerify's per-Miller-loop time is call time / (2 x aggregates).
Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_KEYS = 4096


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def _time(fn, warmup, iters):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters          # ms per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=2048)
    ap.add_argument("--sizes", default="1,16,128")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    import torch
    from pos_evolution_b200.engine import Engine
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    sks = [1 + i for i in range(N_KEYS)]
    assert eng.registry_load(eng.sk_to_pk(sks), np.full(N_KEYS, 32 * 10**9, dtype=np.uint64)).all()
    rng = np.random.default_rng(1)
    result = {"sets": a.sets, "warmup": a.warmup, "iters": a.iters, "aggregate_verify": []}

    for size in [int(x) for x in a.sizes.split(",")]:
        n = a.sets * size
        off = np.arange(0, n + 1, size, dtype=np.uint32)
        signer = rng.integers(0, N_KEYS, size=n).astype(np.uint32)
        msgs = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        sig, st = eng.aggregate(eng.sign([sks[i] for i in signer], np.arange(n, dtype=np.uint32), msgs), off)
        assert (st == 0).all()
        d_signer = torch.as_tensor(signer.astype(np.int32), device=dev)
        d_msgs = torch.as_tensor(msgs, device=dev)
        d_off = torch.as_tensor(off.astype(np.int32), device=dev)
        d_sig = torch.as_tensor(sig, device=dev)
        d_ok = torch.zeros(a.sets, dtype=torch.uint8, device=dev)
        ms = _time(lambda: eng.aggregate_verify_dev(d_signer, d_msgs, d_off, d_sig, d_ok), a.warmup, a.iters)
        assert bool((d_ok == 1).all()), "AggregateVerify rejected an honest set"
        assert eng.guard_flags() == 0
        result["aggregate_verify"].append({"pairs_per_set": size, "ms_per_call": round(ms, 3), "sets_per_s": round(a.sets / ms * 1e3),
                                           "pairs_per_s": round(n / ms * 1e3), "us_per_miller_loop": round(ms * 1e3 / (n + a.sets), 4)})

    # FastAggregateVerify on as many aggregates of one key each: 2 Miller loops + 1 final exponentiation per aggregate
    n = a.sets
    members = rng.integers(0, N_KEYS, size=n).astype(np.uint32)
    msgs = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    sig = eng.sign([sks[i] for i in members], np.arange(n, dtype=np.uint32), msgs)
    d = [torch.as_tensor(x, device=dev) for x in (members.astype(np.int32), np.arange(n + 1, dtype=np.int32), np.ones((n, 1), dtype=np.uint8), msgs, sig)]
    d_ok = torch.zeros(n, dtype=torch.uint8, device=dev)
    ms = _time(lambda: eng.fast_aggregate_verify_dev(*d, d_ok), a.warmup, a.iters)
    assert bool((d_ok == 1).all()), "FastAggregateVerify rejected an honest aggregate"
    result["fast_aggregate_verify"] = {"aggregates": n, "ms_per_call": round(ms, 3), "us_per_miller_loop": round(ms * 1e3 / (2 * n), 4)}
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
