"""Sync-committee aggregate verification on device-resident inputs: b2_sync_aggregate_verify_dev (the committee held on the device with
its precomputed sum; participant or complement sums) beside b2_fast_aggregate_verify_dev fed with the committee's registry indices
repeated for every block, the only way to check these aggregates without the sync-committee entry points.

    python tools/sync_aggregate_bench.py [--blocks 8192] [--participation 1,0.95,0.75,0.5] [--warmup 3] [--iters 10] [--rounds 3]

For each participation level: one 512-key committee, `blocks` blocks with random participation bits and honest signatures (summed secret
keys, signed on the GPU); both paths must give identical verdicts, all 1.  Timing: CUDA events around `iters` calls after `warmup` calls,
the two paths alternating for `rounds` rounds in the same run; the median round is reported.  Prints one JSON line with the card's name
and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE = 512
R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


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
    ap.add_argument("--blocks", type=int, default=8192)
    ap.add_argument("--participation", default="1,0.95,0.75,0.5")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from pos_evolution_b200.engine import Engine
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    sks = [900001 + i for i in range(SIZE)]
    pks = eng.sk_to_pk(sks)
    assert eng.sync_committee_load(pks, SIZE).all()
    assert eng.registry_load(pks, np.full(SIZE, 32 * 10**9, dtype=np.uint64)).all()
    n = a.blocks
    rng = np.random.default_rng(5)
    sk_arr = np.array(sks, dtype=object)
    d_members = torch.as_tensor(np.tile(np.arange(SIZE, dtype=np.int32), n), device=dev)
    d_off = torch.as_tensor((np.arange(n + 1, dtype=np.int64) * SIZE).astype(np.int32), device=dev)
    d_cidx = torch.zeros(n, dtype=torch.int32, device=dev)
    result = {"committee_size": SIZE, "blocks": n, "warmup": a.warmup, "iters": a.iters, "rounds": a.rounds, "levels": []}
    for part in [float(x) for x in a.participation.split(",")]:
        bits = (rng.random((n, SIZE)) < part).astype(np.uint8)
        msgs = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        sums = [int(sk_arr[b.astype(bool)].sum()) % R_ORDER for b in bits]
        assert all(sums)
        sigs = eng.sign(sums, np.arange(n, dtype=np.uint32), msgs)
        rows = np.packbits(bits, axis=1, bitorder="little")
        d_rows, d_msgs, d_sigs = (torch.as_tensor(x, device=dev) for x in (rows, msgs, sigs))
        ok_sync = torch.zeros(n, dtype=torch.uint8, device=dev)
        ok_fav = torch.zeros(n, dtype=torch.uint8, device=dev)
        sync = lambda: eng.sync_aggregate_verify_dev(d_cidx, d_rows, d_msgs, d_sigs, ok_sync)            # noqa: E731
        fav = lambda: eng.fast_aggregate_verify_dev(d_members, d_off, d_rows, d_msgs, d_sigs, ok_fav)     # noqa: E731
        t_sync, t_fav = [], []
        for _ in range(a.rounds):
            t_sync.append(_time(sync, a.warmup, a.iters))
            t_fav.append(_time(fav, a.warmup, a.iters))
        assert torch.equal(ok_sync, ok_fav) and bool((ok_sync == 1).all()), "verdicts differ or an honest block was rejected"
        assert eng.guard_flags() == 0
        ms_s, ms_f = float(np.median(t_sync)), float(np.median(t_fav))
        result["levels"].append({"participation": part, "mean_participants": round(float(bits.sum(axis=1).mean()), 1),
                                 "sync_ms_per_call": round(ms_s, 3), "fast_aggregate_verify_ms_per_call": round(ms_f, 3),
                                 "sync_us_per_block": round(ms_s * 1e3 / n, 3), "speedup": round(ms_f / ms_s, 3),
                                 "sync_ms_rounds": [round(x, 3) for x in t_sync], "fav_ms_rounds": [round(x, 3) for x in t_fav]})
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
