"""Where bls.Aggregate's time goes, per kernel: torch.profiler's device times of k_g2_decompress, k_g2_segment_sum and k_g2_finish
inside eng.aggregate_dev on bench.py's 2^20 individual signatures (2 048 segments of 512), plus the CUDA-event time of the whole
call.  Prints one JSON line with the card's name and power limit beside the numbers.  B2_LIB selects another build of the library
(an A/B of two trees).

    python tools/decompress_profile.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from pos_evolution_b200 import spec as PS  # noqa: E402
from pos_evolution_b200.engine import Engine  # noqa: E402

KERNELS = ("k_g2_decompress", "k_g2_segment_sum", "k_g2_finish")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "max_sm_mhz": int(q[2])} if len(q) == 3 else {"name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    dev = torch.device("cuda", 0)
    d_sigs = torch.as_tensor(W["sigs"], device=dev)
    d_off = torch.as_tensor(W["off"].astype(np.int32), device=dev)
    n_agg = len(W["off"]) - 1
    out = torch.zeros((n_agg, 96), dtype=torch.uint8, device=dev)
    st = torch.zeros(n_agg, dtype=torch.int32, device=dev)
    run = lambda: eng.aggregate_dev(d_sigs, d_off, out, st)           # noqa: E731
    run()                                                               # warm-up: scratch buffers, module load
    torch.cuda.synchronize()
    ev = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ev.append(e0.elapsed_time(e1))
    assert int((st != 0).sum().item()) == 0, "an aggregate failed"
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            run()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key and e.count:
                per[k] = {"mean": e.self_device_time_total / e.count / 1e3, "launches": e.count}
    res = {"card": card(), "signatures": int(W["off"][-1]), "segments": n_agg, "reps": args.reps,
           "aggregate_dev_ms": {"mean": sum(ev) / len(ev), "min": min(ev), "max": max(ev)},
           "kernel_ms": per, "agg_sig0": bytes(out[0].cpu().numpy()).hex()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
