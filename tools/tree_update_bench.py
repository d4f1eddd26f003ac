"""Changing the fork-choice block tree on the device (b2_tree_add / _prune / _set_viable) against reloading it (b2_tree_load, and
b2_latest_messages_load after a prune), at 2^20 validators on a scenarios.fork_tree(10 000) tree.  Every call is synchronous, so a host
clock around it is its time; each case reports the median and range over repeated rounds.  The add / set_viable / prune cases start
from a fresh tree_load, so they include the first call's allocation of the change scratch; `add1_get_head_steady` appends one block per
round to the same tree (the per-slot case).  A separate torch.profiler pass gives the kernel times per call, and the Spec case times
get_head after one new block at 2^16 validators with the incremental mirror against the full re-upload.  Prints one JSON line with the
card's name and power limit.

    python tools/tree_update_bench.py [--rounds 15] [--validators 1048576] [--blocks 10000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import scenarios  # noqa: E402
from pos_evolution_b200.engine import Engine  # noqa: E402

INF_PK = bytes([0xC0]) + bytes(47)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, rounds, setup=None):
    ts = []
    for _ in range(rounds):
        if setup:
            setup()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return {"median_ms": round(ts[len(ts) // 2], 4), "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4)}


def profile(e, reset, add, root, rounds):
    """CUDA kernel time per call of each kernel of the tree calls, from one torch.profiler pass"""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    reset()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            add(1)
        add(1024)
        e.tree_prune(root)
        torch.cuda.synchronize()
    calls = {"k_tree_insert_cta": rounds + 1, "k_tree_rank_old": rounds + 1, "k_tree_rank_new": rounds + 1, "k_tree_emit": rounds + 2,
             "k_tree_prune": 1, "k_lmd_remap": 1}
    out = {}
    for ev in prof.key_averages():
        for k, c in calls.items():
            if k in ev.key:
                total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                out[k] = round(out.get(k, 0) + total / c, 2)
    return out


def spec_case(rounds):
    """Spec.get_head after one new block, 2^16 validators on a 1 000-block store: the incremental mirror against the full re-upload"""
    from pos_evolution_b200 import spec as PS
    from test_host_logic import _mirror_world
    store, state, rb, slot = _mirror_world(PS, n_val=1 << 16, n_blocks=1000)
    res = {}
    for inc in (True, False):
        sp = PS.Spec(PS.MINIMAL, engine=Engine(0), incremental_tree=inc)
        sp.get_head(store)
        ts = []
        for i in range(rounds):
            parent = sp.get_head(store)
            root = (0x5000 + 100 * inc + i).to_bytes(2, "big") * 16
            store.blocks[root] = PS.BeaconBlock(store.blocks[parent].slot + 1, parent)
            store.block_states[root] = store.block_states[parent]
            t0 = time.perf_counter()
            sp.get_head(store)
            ts.append((time.perf_counter() - t0) * 1e3)
        ts.sort()
        res["incremental" if inc else "full_reload"] = {"median_ms": round(ts[len(ts) // 2], 3), "min_ms": round(ts[0], 3), "max_ms": round(ts[-1], 3),
                                                        "store_uploads": sp.stats["store_uploads"], "tree_adds": sp.stats["tree_adds"]}
        sp.engine.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--validators", type=int, default=1 << 20)
    ap.add_argument("--blocks", type=int, default=10_000)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    n_val, n = a.validators, a.blocks
    parent, slot, roots, viable = scenarios.fork_tree(n + 1024 * (a.rounds + 2) + 64 * (a.rounds + 2))
    e = Engine(0)
    e.registry_load(np.frombuffer(INF_PK * n_val, dtype=np.uint8).reshape(n_val, 48), (rng.integers(1, 33, n_val) * 10**9).astype(np.uint64))
    epoch = rng.integers(1, 100, n_val).astype(np.uint64)
    block = rng.integers(0, n, n_val).astype(np.uint32)
    has = np.ones(n_val, dtype=np.uint8)
    eq = np.zeros(n_val, dtype=np.uint8)
    out = {"card": card(), "validators": n_val, "blocks": n, "rounds": a.rounds}

    def reset():
        e.tree_load(parent[:n], slot[:n], roots[:n], viable[:n])
        e.latest_messages_load(epoch, block, has, eq)
        e.get_head(0)

    def add(k):
        m = e.tree_size()
        e.tree_add(parent[m:m + k], slot[m:m + k], roots[m:m + k], viable[m:m + k])

    reset()
    out["add1_get_head_steady"] = timed(lambda: (add(1), e.get_head(0)), 4 * a.rounds)
    reset()
    out["add1_get_head"] = timed(lambda: (add(1), e.get_head(0)), a.rounds, reset)
    out["load_n1_get_head"] = timed(lambda: (e.tree_load(parent[:n + 1], slot[:n + 1], roots[:n + 1], viable[:n + 1]), e.get_head(0)), a.rounds)
    out["add32"] = timed(lambda: add(32), a.rounds, reset)
    out["add1024"] = timed(lambda: add(1024), a.rounds, reset)
    leaf = n - 1
    out["set_viable1"] = timed(lambda: e.tree_set_viable([leaf], [1]), a.rounds, reset)
    size = np.ones(n, dtype=np.int64)
    for b in range(n - 1, 0, -1):
        size[parent[b]] += size[b]
    root = int(np.argmin(np.abs(size - 2 * n // 3)))
    maps = []
    out["prune_two_thirds"] = timed(lambda: maps.append(e.tree_prune(root)), a.rounds, reset)
    mp = maps[-1]
    kept = mp != 0xFFFFFFFF
    k_parent = mp[parent[:n][kept]]
    k_parent[0] = 0
    k_block = np.where(block < n, mp[np.minimum(block, n - 1)], block)
    out["kept_blocks"] = int(kept.sum())
    out["load_pruned_plus_lmd_load"] = timed(lambda: (e.tree_load(k_parent, slot[:n][kept], roots[:n][kept], viable[:n][kept]),
                                                      e.latest_messages_load(epoch, k_block, has, eq)), a.rounds)
    reset()
    e.tree_prune(root)
    e_b = e.latest_messages_read()[1]
    assert np.array_equal(e_b, k_block), "device re-map differs from the host compaction"
    out["kernels_us_per_call"] = profile(e, reset, add, root, a.rounds)
    e.close()
    out["spec_2e16"] = spec_case(a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
