"""hash_tree_root of the beacon state's large fields on the GPU (b2_ssz_*) at mainnet size: a registry of 2^20 validators.

    python tools/state_root_bench.py [--warmup 2] [--iters 5] [--rounds 5] [--skip-oracle]

Workloads: ssz_validators_load of 2^20 random records (a full rebuild), ssz_validators_update of k = 64, 4 096 and 65 536 random records
(sorted indices; the update workloads on both sides of where a rebuild could win), ssz_chunks_root of 2^20 balances (List[Gwei, 2^40])
and of 65 536 randao mixes (Vector[Bytes32, 65536]).  Each call is timed with CUDA events around the synchronous call (uploads and the
32-byte download included), median and range over `rounds` rounds of `iters` calls after `warmup` calls.  One torch.profiler pass splits
each workload into kernel time and host-to-device copy time.  Node hashes are counted from the shapes: 8 per validator leaf, one per
distinct inner node on the re-hashed paths, the zero-padding chain to the limit depth and the length mix-in.  The hashlib oracle
(tests/ssz_oracle.py) times the same roots on the CPU, and every GPU root is checked against it.  Prints one JSON line with the card's
name and power limit, read in the same run.  Writes nothing."""
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

N_VAL, N_MIXES, REG_DEPTH = 1 << 20, 1 << 16, 40
UPDATE_K = (64, 4096, 65536)


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


def tree_hashes(n_leaves: int, idx=None) -> int:
    """inner node hashes of a heap over C = next_pow2(n_leaves) leaves: all of them, or those on the paths of the leaves idx"""
    C = 1 << max(n_leaves - 1, 0).bit_length()
    if idx is None:
        return C - 1
    total, nodes = 0, np.asarray(idx, dtype=np.int64) + C
    while C > 1:
        nodes = np.unique(nodes >> 1)
        total += len(nodes)
        C >>= 1
    return total


def root_hashes(n_leaves: int, depth: int, mix_in: bool) -> int:
    """the serial finish: zero-padding from depth log2 C to `depth`, then the length mix-in"""
    return depth - max(n_leaves - 1, 0).bit_length() + int(mix_in)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-oracle", action="store_true", help="skip the CPU oracle (its 2^20-validator root takes tens of seconds)")
    a = ap.parse_args()
    import torch
    import ssz_oracle as O
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.spec import MAINNET, _chunk_depth

    card, power = _card()
    eng = Engine(0)
    rng = np.random.default_rng(1)
    rec = rng.integers(0, 256, size=(N_VAL, 121), dtype=np.uint8)
    rec[:, 88] &= 1
    balances = rng.integers(16 * 10**9, 33 * 10**9, size=N_VAL, dtype=np.uint64)
    mixes = rng.integers(0, 256, size=(N_MIXES, 32), dtype=np.uint8)
    bal_depth, mix_depth = _chunk_depth(MAINNET.VALIDATOR_REGISTRY_LIMIT, 8), _chunk_depth(MAINNET.EPOCHS_PER_HISTORICAL_VECTOR, 32)
    updates = {}
    for k in UPDATE_K:
        idx = np.sort(rng.choice(N_VAL, size=k, replace=False)).astype(np.uint32)
        new = rng.integers(0, 256, size=(k, 121), dtype=np.uint8)
        new[:, 88] &= 1
        updates[k] = (idx, new)

    # each workload: (call, node hashes, bytes uploaded)
    work = {"validators_load": (lambda: eng.ssz_validators_load(rec), 8 * N_VAL + tree_hashes(N_VAL) + root_hashes(N_VAL, REG_DEPTH, True),
                                rec.nbytes)}
    for k, (idx, new) in updates.items():
        # alternating between the new and the original records keeps every call an update of k changed leaves
        state = {"flip": False}

        def call(idx=idx, new=new, old=rec[idx], state=state):
            state["flip"] = not state["flip"]
            return eng.ssz_validators_update(idx, new if state["flip"] else old)

        work["validators_update_%d" % k] = (call, 8 * k + tree_hashes(N_VAL, idx) + root_hashes(N_VAL, REG_DEPTH, True), idx.nbytes + new.nbytes)
    n_bal_chunks = N_VAL * 8 // 32
    work["balances_root"] = (lambda: eng.ssz_chunks_root(balances, bal_depth, N_VAL),
                             tree_hashes(n_bal_chunks) + root_hashes(n_bal_chunks, bal_depth, True), balances.nbytes)
    work["randao_mixes_root"] = (lambda: eng.ssz_chunks_root(mixes, mix_depth), tree_hashes(N_MIXES) + root_hashes(N_MIXES, mix_depth, False),
                                 mixes.nbytes)

    # correctness first: the GPU roots against the oracle (or against each other without it)
    eng.ssz_validators_load(rec)
    roots = {"validators_load": eng.ssz_validators_load(rec), "balances_root": eng.ssz_chunks_root(balances, bal_depth, N_VAL),
             "randao_mixes_root": eng.ssz_chunks_root(mixes, mix_depth)}
    cpu_s = {}
    if not a.skip_oracle:
        t = time.perf_counter()
        want = O.records_root([bytes(r) for r in rec], MAINNET.VALIDATOR_REGISTRY_LIMIT)
        cpu_s["validators_load"] = time.perf_counter() - t
        assert roots["validators_load"] == want
        t = time.perf_counter()
        assert roots["balances_root"] == O.basic_list_root([int(b) for b in balances], 8, MAINNET.VALIDATOR_REGISTRY_LIMIT)
        cpu_s["balances_root"] = time.perf_counter() - t
        t = time.perf_counter()
        assert roots["randao_mixes_root"] == O.roots_vector_root([bytes(m) for m in mixes])
        cpu_s["randao_mixes_root"] = time.perf_counter() - t
    for k, (idx, new) in updates.items():
        upd = eng.ssz_validators_update(idx, new)
        fresh = rec.copy()
        fresh[idx] = new
        assert upd == eng.ssz_validators_load(fresh), k      # an update equals a rebuild of the same records
        eng.ssz_validators_load(rec)

    eng.ssz_validators_load(rec)
    res = {}
    for name, (call, hashes, up_bytes) in work.items():
        for _ in range(a.warmup):
            call()
        times = []
        for _ in range(a.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / a.iters)
        res[name] = {"ms": round(float(np.median(times)), 4), "ms_range": [round(min(times), 4), round(max(times), 4)], "node_hashes": int(hashes),
                     "upload_bytes": int(up_bytes)}
        if name in cpu_s:
            res[name]["cpu_oracle_s"] = round(cpu_s[name], 2)

    from torch.profiler import ProfilerActivity, profile
    for name, (call, hashes, _) in work.items():
        eng.ssz_validators_load(rec)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                call()
            torch.cuda.synchronize()
        kern = copy = 0.0
        per_kernel = {}
        for ev in prof.key_averages():
            if ev.device_type.name != "CUDA" or not ev.count:
                continue
            t = (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) / a.iters / 1e3
            if "Memcpy HtoD" in ev.key:
                copy += t
            elif "k_ssz" in ev.key:
                kern += t
                per_kernel[ev.key.split("(")[0].replace("void ", "").replace("b2::", "")] = round(t, 4)
        res[name].update({"kernel_ms": round(kern, 4), "h2d_ms": round(copy, 4), "kernels_ms": per_kernel,
                          "node_hashes_per_s_kernel": float("%.4g" % (hashes / (kern * 1e-3))) if kern else None})
    eng.close()
    print(json.dumps({"card": card, "power_limit": power, "validators": N_VAL, "results": res}))


if __name__ == "__main__":
    main()
