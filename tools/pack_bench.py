"""Block packing (b2_pack_attestations / _dev) at mainnet size: 2^20 validators, both includable epochs with 2 048 committees of 512
each (4 096 committees), per committee two votes (head variants) with `--aggs` overlapping aggregates at high participation and
`--singles` single-bit attestations, participation prefilled for 30 % of the validators, MAX_ATTESTATIONS = 128 picks.  Signatures are
made by linearity, as bench.py does (one Sign per candidate with a per-candidate scalar standing for the sum of its signers' keys).

    python tools/pack_bench.py [--aggs 4] [--singles 8] [--warmup 2] [--iters 10] [--rounds 3]

Times the host form (host clock around the synchronous call, uploads and downloads included) and the _dev form (CUDA events around
the enqueued call on device arrays), median and range over `rounds` rounds of `iters` calls; the kernel breakdown from one
torch.profiler pass; and the CPU per-committee reference (tests/pack_oracle.py) on the same pool, whose picks the GPU must equal.
Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_VAL, PER_TABLE, CSIZE, MAX_OUT = 1 << 20, 2048, 512, 128


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


def make_pool(aggs, singles, seed=1):
    rng = np.random.default_rng(seed)
    eff = rng.choice([16, 24, 31, 32, 32, 32, 32], size=N_VAL).astype(np.uint64) * np.uint64(10**9)
    part = [(rng.integers(0, 8, size=N_VAL) * (rng.random(N_VAL) < 0.3)).astype(np.uint8) for _ in range(2)]
    members = np.concatenate([rng.permutation(N_VAL) for _ in range(2)]).astype(np.uint32)
    K = 2 * PER_TABLE
    off = (np.arange(K + 1, dtype=np.int64) * CSIZE).astype(np.uint32)
    table = np.repeat(np.arange(2, dtype=np.uint8), PER_TABLE)
    per = 2 * (aggs + singles)
    comm = np.repeat(np.arange(K, dtype=np.uint32), per)
    vote = np.tile(np.repeat(np.arange(2, dtype=np.uint32), aggs + singles), K)
    data = comm * 2 + vote
    vote_mask = np.where(np.arange(2 * K) % 2 == 0, 7, 3).astype(np.uint8)         # the head variant misses the head flag
    is_single = np.tile(np.r_[np.zeros(aggs, bool), np.ones(singles, bool)], 2 * K)
    rows = rng.random((len(comm), CSIZE)) < np.where(is_single, 0.0, rng.choice([0.8, 0.9, 0.95], size=len(comm)))[:, None]
    single_bit = rng.integers(0, CSIZE, size=len(comm))
    rows[np.nonzero(is_single)[0], single_bit[is_single]] = True
    bits = np.packbits(rows, axis=1, bitorder="little")
    return {"members": members, "off": off, "table": table, "comm": comm, "data": data.astype(np.uint32), "mask": vote_mask[data], "bits": bits,
            "ok": [True] * len(comm), "eff": eff, "part": part, "inc": 10**9, "per_inc": 1000, "max_out": MAX_OUT}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--aggs", type=int, default=4)
    ap.add_argument("--singles", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import pack_oracle as PO
    from oracle.bls12_381 import G1, g1_compress
    from pos_evolution_b200.engine import Engine
    if not torch.cuda.is_available():
        raise SystemExit("pack_bench needs a GPU")
    card, power = _card()
    pool = make_pool(a.aggs, a.singles)
    C = len(pool["comm"])
    eng = Engine(0)
    eng.registry_load(np.tile(np.frombuffer(g1_compress(G1), dtype=np.uint8), (N_VAL, 1)), pool["eff"])
    eng.participation_load(0, pool["part"][0])
    eng.participation_load(1, pool["part"][1])
    msgs = np.frombuffer(b"".join(d.to_bytes(4, "little") + bytes(28) for d in range(2 * 2 * PER_TABLE)), dtype=np.uint8).reshape(-1, 32)
    sigs = eng.sign(list(range(1, C + 1)), pool["data"], msgs)
    args = (pool["members"], pool["off"], pool["table"], pool["comm"], pool["data"], pool["mask"], pool["bits"], sigs, MAX_OUT, pool["inc"],
            pool["per_inc"])

    t0 = time.perf_counter()
    ref = PO.pack_per_committee(pool)
    cpu_s = time.perf_counter() - t0
    res = eng.pack_attestations(*args)
    got = [(int(res.committee[o]), int(res.data[o]), int.from_bytes(res.bits[o].tobytes(), "little"), int(res.numerator[o]),
            tuple(int(x) for x in res.src[res.src_off[o]:res.src_off[o + 1]])) for o in range(len(res.committee))]
    assert got == ref, "GPU packing differs from the per-committee reference"

    host = []
    for _ in range(a.warmup):
        eng.pack_attestations(*args)
    for _ in range(a.rounds):
        t = time.perf_counter()
        for _ in range(a.iters):
            eng.pack_attestations(*args)
        host.append((time.perf_counter() - t) / a.iters * 1e3)

    dev = torch.device("cuda", 0)
    i32 = lambda x: torch.as_tensor(np.ascontiguousarray(x, dtype=np.uint32).view(np.int32), device=dev)    # noqa: E731
    u8 = lambda x: torch.as_tensor(np.ascontiguousarray(x, dtype=np.uint8), device=dev)                    # noqa: E731
    dins = (i32(pool["members"]), i32(pool["off"]), u8(pool["table"]), i32(pool["comm"]), i32(pool["data"]), u8(pool["mask"]), u8(pool["bits"]),
            u8(sigs))
    outs = (torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(MAX_OUT, dtype=torch.int32, device=dev),
            torch.zeros(MAX_OUT, dtype=torch.int32, device=dev), torch.zeros((MAX_OUT, CSIZE // 8), dtype=torch.uint8, device=dev),
            torch.zeros((MAX_OUT, 96), dtype=torch.uint8, device=dev), torch.zeros(MAX_OUT, dtype=torch.int64, device=dev),
            torch.zeros(MAX_OUT + 1, dtype=torch.int32, device=dev), torch.zeros(C, dtype=torch.int32, device=dev),
            torch.zeros(C, dtype=torch.uint8, device=dev))

    def dev_call():
        eng.pack_attestations_dev(*dins, MAX_OUT, pool["inc"], pool["per_inc"], *outs)

    for _ in range(a.warmup):
        dev_call()
    torch.cuda.synchronize()
    assert np.array_equal(outs[4][:len(got)].cpu().numpy(), res.signature) and int(outs[0].item()) == len(got)
    devt = []
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            dev_call()
        e1.record()
        torch.cuda.synchronize()
        devt.append(e0.elapsed_time(e1) / a.iters)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            dev_call()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ev.count:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            kernels[ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("b2::", "")] = round(t / 3 / 1e3, 4)
    eng.close()
    med = lambda x: round(float(np.median(x)), 3)     # noqa: E731
    print(json.dumps({"card": card, "power_limit": power, "validators": N_VAL, "committees": 2 * PER_TABLE, "candidates": C,
                      "folded_picks": len(got), "host_ms": med(host), "host_ms_range": [round(min(host), 3), round(max(host), 3)],
                      "dev_ms": med(devt), "dev_ms_range": [round(min(devt), 3), round(max(devt), 3)], "kernels_ms": kernels,
                      "cpu_reference_s": round(cpu_s, 2)}))


if __name__ == "__main__":
    main()
