"""What one slot of sync committee contributions costs: 2^20 validators, the mainnet committee (512 positions over 4 subnets), aggregators
selected by their own selection proofs (TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE = 16), contributions over 2 roots signed through
Engine.sign with the arithmetic-progression keys.

    python tools/sync_contributions_bench.py [--rounds 7]
    python tools/sync_contributions_bench.py --profile     # one torch.profiler pass per load: the split over the call's kernels

Two loads: the expected one (16 aggregators per subnet, 64 items) and 1 024 items, where the expected load is followed by re-sent items,
subsets of them and items of the same aggregators on the other root.  Reported per load:
  device_ms   device time of one Engine.sync_contribution_and_proof_intake_dev call (CUDA events, median and range over the rounds);
  host_s      wall time of the same checks through the existing synchronous batched calls: Engine.aggregate_verify over the 2n single-key
              sets, Engine.fast_aggregate_verify over the contributions, the list-order rules in numpy, and Engine.aggregate per root (the
              wire decode and the SSZ roots are not counted).
The two paths' aggregate signatures are checked equal.  Prints one JSON line with the card's name and power limit, read in the same run.
Writes nothing."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402
import sync_contributions_oracle as C  # noqa: E402
from epoch_discount_bench import _card  # noqa: E402
from sync_messages_bench import _h  # noqa: E402

SIZE, COUNT, SLOT, TARGET = 512, 4, 123456, 16
SUB = SIZE // COUNT


def keys(eng):
    n = bench.N_VAL
    sk0 = int.from_bytes(_h(b"b200pos/sk0"), "big") % (bench.R_ORDER >> 1) or 1
    delta = int.from_bytes(_h(b"b200pos/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), dtype=np.uint32).reshape(n, 8)
    eng.registry_load(eng.sk_to_pk(sk8), np.full(n, 32 * 10**9, np.uint64))
    return lambda v: sk0 + int(v) * delta


def sign(eng, sks, msgs):
    m = np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32)
    return [bytes(x) for x in eng.sign([k % bench.R_ORDER for k in sks], np.arange(len(msgs), dtype=np.uint32), m)]


def slot_items(eng, sk, n_items, rng):
    """(wires, plan, pv, domains, roots): 16 selected aggregators per subnet, one contribution each, then re-sends, subsets and the other
    root up to n_items"""
    pv = rng.choice(bench.N_VAL, SIZE, replace=False).astype(np.uint32)
    domains = _h(b"sync-domain") + _h(b"selection-domain") + _h(b"cap-domain")
    roots = [_h(b"contribution-root" + bytes([k])) for k in range(2)]
    pairs = [(int(pv[p]), p // SUB) for p in range(SIZE)]
    proofs = sign(eng, [sk(v) for v, s in pairs], [C.signing_root(C.selection_data_root(SLOT, s), domains[32:64]) for v, s in pairs])
    chosen = {s: [] for s in range(COUNT)}
    for (v, s), p in zip(pairs, proofs):
        if C.is_aggregator(p, SUB, TARGET) and len(chosen[s]) < 16 and v not in chosen[s]:
            chosen[s].append(v)
    plan = [(v, s, j % 2, [bool(x) for x in rng.random(SUB) < 0.8]) for s in range(COUNT) for j, v in enumerate(chosen[s])]
    base = list(plan)
    while len(plan) < n_items:
        v, s, k, bits = base[int(rng.integers(0, len(base)))]
        kind = int(rng.integers(0, 3))
        if kind == 1:
            bits = [b and rng.random() < 0.7 for b in bits]
        elif kind == 2:
            k = 1 - k
        plan.append((v, s, k, bits if any(bits) else [True] + bits[1:]))
    plan = plan[:n_items]
    prf = sign(eng, [sk(v) for v, s, k, b in plan], [C.signing_root(C.selection_data_root(SLOT, s), domains[32:64]) for v, s, k, b in plan])
    sig = sign(eng, [sum(sk(pv[s * SUB + i]) for i, x in enumerate(b) if x) for v, s, k, b in plan],
               [C.signing_root(roots[k], domains[:32]) for v, s, k, b in plan])
    caps = [C.signing_root(C.contribution_and_proof_root(v, SLOT, roots[k], s, C.pack(b), sig[a], prf[a]), domains[64:96])
            for a, (v, s, k, b) in enumerate(plan)]
    out = sign(eng, [sk(v) for v, s, k, b in plan], caps)
    wires = [C.encode(v, SLOT, roots[k], s, b, sig[a], prf[a], out[a]) for a, (v, s, k, b) in enumerate(plan)]
    return wires, plan, pv, domains, roots, (prf, sig, caps, out)


def host_path(eng, plan, pv, domains, roots, signed):
    """the existing batched calls: AggregateVerify of the 2n single-key sets, FastAggregateVerify of the contributions, the list-order
    rules in numpy, then bls.Aggregate of each root's best contributions"""
    prf, sig, caps, out = signed
    n = len(plan)
    v = np.array([x[0] for x in plan], np.uint32)
    s = np.array([x[1] for x in plan], np.uint32)
    k = np.array([x[2] for x in plan], np.uint32)
    bits = np.array([x[3] for x in plan], bool)
    sel = np.frombuffer(b"".join(C.signing_root(C.selection_data_root(SLOT, int(x)), domains[32:64]) for x in s), np.uint8).reshape(n, 32)
    msgs = np.stack([sel, np.frombuffer(b"".join(caps), np.uint8).reshape(n, 32)], 1).reshape(2 * n, 32)
    sigs = np.stack([np.frombuffer(b"".join(prf), np.uint8).reshape(n, 96), np.frombuffer(b"".join(out), np.uint8).reshape(n, 96)], 1).reshape(2 * n, 96)
    av = eng.aggregate_verify(np.repeat(v, 2), np.arange(2 * n + 1, dtype=np.uint32), msgs, sigs).reshape(n, 2)
    members = np.concatenate([pv[x * SUB:(x + 1) * SUB] for x in s])
    rows = np.packbits(bits, axis=1, bitorder="little")
    sync = np.frombuffer(b"".join(C.signing_root(roots[x], domains[:32]) for x in k), np.uint8).reshape(n, 32)
    csig = np.frombuffer(b"".join(sig), np.uint8).reshape(n, 96)
    fav = eng.fast_aggregate_verify(members, np.arange(n + 1, dtype=np.uint32) * SUB, rows, sync, csig)
    acc = {}          # (root, subnet) -> accepted bit rows; (aggregator, subnet) seen
    seen, best = set(), {}
    for a in range(n):
        key = (int(k[a]), int(s[a]))
        if any(not (bits[a] & ~b).any() for b in acc.get(key, [])) or (int(v[a]), int(s[a])) in seen:
            continue
        if av[a, 0] and av[a, 1] and fav[a]:
            acc.setdefault(key, []).append(bits[a])
            seen.add((int(v[a]), int(s[a])))
            c = int(bits[a].sum())
            if key not in best or c > best[key][0]:
                best[key] = (c, a)
    src, off = [], [0]
    for r in range(2):
        src += [best[(r, x)][1] for x in range(COUNT) if (r, x) in best]
        off.append(len(src))
    agg, _ = eng.aggregate(csig[src], np.array(off, np.uint32))
    return agg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    sk = keys(eng)
    dev = torch.device("cuda", 0)
    out = {"tool": "sync_contributions_bench", "validators": bench.N_VAL, "committee_size": SIZE}
    for n_items in (64, 1024):
        wires, plan, pv, domains, roots, signed = slot_items(eng, sk, n_items, np.random.default_rng(11 + n_items))
        woff = np.cumsum([0] + [len(w) for w in wires]).astype(np.int32)
        d = [torch.as_tensor(np.frombuffer(b"".join(wires), np.uint8).copy(), device=dev), torch.as_tensor(woff, device=dev),
             torch.as_tensor(pv.astype(np.int32), device=dev)]
        res, nr = eng.sync_contribution_and_proof_intake_dev(*d, COUNT, SLOT, domains, TARGET, trim=False)      # warm-up
        torch.cuda.synchronize()
        status = res.status.cpu().numpy()
        assert int(nr.cpu()[0]) == 2 and set(status.tolist()) <= {0, 8, 9}, "every item verifies; the rest are list-order IGNOREs"
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                eng.sync_contribution_and_proof_intake_dev(*d, COUNT, SLOT, domains, TARGET, out=(res, nr), trim=False)
                torch.cuda.synchronize()
            split = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                    split[ev.key] = round(ev.device_time_total / 1000.0, 3)
            out["profile_ms_%d_items" % n_items] = dict(sorted(split.items(), key=lambda kv: -kv[1]))
            continue
        times = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.sync_contribution_and_proof_intake_dev(*d, COUNT, SLOT, domains, TARGET, out=(res, nr), trim=False)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        host = []
        for _ in range(max(1, args.rounds // 2)):
            t0 = time.perf_counter()
            agg = host_path(eng, plan, pv, domains, roots, signed)
            host.append(time.perf_counter() - t0)
        got = res.agg_sigs.cpu().numpy()
        first = {}
        for a in range(len(plan)):
            if status[a] == 0 and plan[a][2] not in first:
                first[plan[a][2]] = int(res.root_id[a].item())
        assert all(np.array_equal(got[first[r]], agg[r]) for r in range(2)), "aggregate signatures differ"
        out["%d_items" % n_items] = {"accepted": int((status == 0).sum()), "device_ms": round(float(np.median(times)), 3),
                                     "device_ms_range": [round(min(times), 3), round(max(times), 3)],
                                     "host_s": round(float(np.median(host)), 4), "host_s_range": [round(min(host), 4), round(max(host), 4)]}
    out["gpu"], out["power_limit"] = _card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
