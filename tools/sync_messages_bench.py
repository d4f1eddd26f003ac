"""What one slot of sync committee messages costs: 2^20 validators, the mainnet committee (512 positions, a few validators holding two),
one message per (validator, subnet) of the committee plus 5 % duplicates, signed over 1 or 2 roots through Engine.sign with the
arithmetic-progression keys.

    python tools/sync_messages_bench.py [--rounds 7]
    python tools/sync_messages_bench.py --profile     # one torch.profiler pass per root count: the split over the call's kernels

Reported per root count:
  device_ms   device time of one Engine.sync_committee_messages_dev call (CUDA events, median and range over the rounds);
  host_s      wall time of the same work through the existing synchronous batched calls: Engine.aggregate_verify over the messages as
              single-key sets, the seen rule and the grouping by (root, subnet) in numpy, and Engine.aggregate over the contributions and
              the aggregates (the per-message wire decode and subnet check are not counted).
The two paths' aggregate signatures are checked equal.  Prints one JSON line with the card's name and power limit, read in the same run.
Writes nothing."""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402
from epoch_discount_bench import _card  # noqa: E402

SIZE, COUNT, SLOT = 512, 4, 123456


def _h(b):
    return hashlib.sha256(b).digest()


def world(eng):
    n = bench.N_VAL
    sk0 = int.from_bytes(_h(b"b200pos/sk0"), "big") % (bench.R_ORDER >> 1) or 1
    delta = int.from_bytes(_h(b"b200pos/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), dtype=np.uint32).reshape(n, 8)
    eng.registry_load(eng.sk_to_pk(sk8), np.full(n, 32 * 10**9, np.uint64))
    return sk8


def messages(eng, sk8, n_roots, rng):
    """(wire, woff, subnet, position_validator, domain, roots): every (validator, subnet) once, 5 % of them again later"""
    pv = rng.choice(bench.N_VAL, SIZE, replace=False).astype(np.uint32)
    pv[SIZE // 2 + 1::37] = pv[1:SIZE // 2:37][:len(pv[SIZE // 2 + 1::37])]      # a few validators in two subnets
    sub = SIZE // COUNT
    pairs = sorted({(int(pv[p]), p // sub) for p in range(SIZE)})
    items = [(v, s, int(rng.integers(0, n_roots))) for v, s in pairs]
    items += [items[i] for i in rng.choice(len(items), len(items) // 20, replace=False)]
    roots = [_h(b"sync-root" + bytes([k])) for k in range(n_roots)]
    domain = _h(b"sync-domain")
    msgs = np.frombuffer(b"".join(_h(r + domain) for r in roots), np.uint8).reshape(n_roots, 32)
    sigs = eng.sign(sk8[[v for v, _, _ in items]], [k for _, _, k in items], msgs)
    wire = b"".join(SLOT.to_bytes(8, "little") + roots[k] + v.to_bytes(8, "little") + sigs[a].tobytes() for a, (v, s, k) in enumerate(items))
    woff = np.arange(len(items) + 1, dtype=np.uint32) * 144
    return wire, woff, np.array([s for _, s, _ in items], np.uint32), pv, domain, roots, msgs, items


def host_path(eng, items, pv, msgs, sigs, n_roots):
    """the existing batched calls: verify every message, seen rule and grouping in numpy, then bls.Aggregate per contribution and root"""
    n = len(items)
    v = np.array([x[0] for x in items], np.uint32)
    s = np.array([x[1] for x in items], np.uint32)
    k = np.array([x[2] for x in items], np.uint32)
    ok = eng.aggregate_verify(v, np.arange(n + 1, dtype=np.uint32), msgs[k], sigs)
    key = v.astype(np.uint64) * COUNT + s
    first = np.full(n, False)
    good = np.flatnonzero(ok)
    _, idx = np.unique(key[good], return_index=True)
    first[good[idx]] = True                                  # the first verified item of each (validator, subnet)
    acc = {(int(v[a]), int(s[a])): a for a in np.flatnonzero(first)}
    sub = SIZE // COUNT
    src, seg = [], [0]
    for r in range(n_roots):
        for sc in range(COUNT):
            for p in range(sc * sub, (sc + 1) * sub):
                a = acc.get((int(pv[p]), sc))
                if a is not None and k[a] == r:
                    src.append(a)
            seg.append(len(src))
    eng.aggregate(sigs[src], np.array(seg, np.uint32))      # the contributions
    agg_off = np.array(seg[::COUNT], np.uint32)
    agg, _ = eng.aggregate(sigs[src], agg_off)
    return agg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    sk8 = world(eng)
    dev = torch.device("cuda", 0)
    out = {"tool": "sync_messages_bench", "validators": bench.N_VAL, "committee_size": SIZE}
    for n_roots in (1, 2):
        wire, woff, subnet, pv, domain, roots, msgs, items = messages(eng, sk8, n_roots, np.random.default_rng(7 + n_roots))
        d = [torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=dev), torch.as_tensor(woff.astype(np.int32), device=dev),
             torch.as_tensor(subnet.astype(np.int32), device=dev), torch.as_tensor(pv.astype(np.int32), device=dev)]
        res, nr = eng.sync_committee_messages_dev(*d, COUNT, SLOT, domain, trim=False)      # warm-up: module load, scratch allocation
        torch.cuda.synchronize()
        status = res.status.cpu().numpy()
        assert int(nr.cpu()[0]) == n_roots and set(status.tolist()) <= {0, 5}, "every message verifies; the repeats are seen"
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                eng.sync_committee_messages_dev(*d, COUNT, SLOT, domain, out=(res, nr), trim=False)
                torch.cuda.synchronize()
            split = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                    split[ev.key] = round(ev.device_time_total / 1000.0, 3)
            out["profile_ms_%d_roots" % n_roots] = dict(sorted(split.items(), key=lambda kv: -kv[1]))
            continue
        times = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.sync_committee_messages_dev(*d, COUNT, SLOT, domain, out=(res, nr), trim=False)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        sigs = np.frombuffer(wire, np.uint8).reshape(-1, 144)[:, 48:].copy()
        host = []
        for _ in range(max(1, args.rounds // 2)):
            t0 = time.perf_counter()
            agg = host_path(eng, items, pv, msgs, sigs, n_roots)
            host.append(time.perf_counter() - t0)
        # root ids follow first occurrence; the host path numbers roots by index
        first = [int(res.root_id[a].item()) for a in range(len(items))]
        order = {}
        for a, (v, s, k) in enumerate(items):
            if status[a] == 0 and k not in order:
                order[k] = first[a]
        dev_agg = res.agg_sigs.cpu().numpy()
        assert all(np.array_equal(dev_agg[order[k]], agg[k]) for k in range(n_roots)), "aggregate signatures differ"
        out["%d_roots" % n_roots] = {"messages": len(items), "accepted": int((status == 0).sum()),
                                     "device_ms": round(float(np.median(times)), 3),
                                     "device_ms_range": [round(min(times), 3), round(max(times), 3)],
                                     "host_s": round(float(np.median(host)), 4), "host_s_range": [round(min(host), 4), round(max(host), 4)]}
    out["gpu"], out["power_limit"] = _card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
