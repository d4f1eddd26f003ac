"""What the aggregated-attestation intake costs: one epoch of SignedAggregateAndProof gossip at bench.py's size (2^20 validators, 2 048
committees x 512, keys and committees from bench.build_world), with the aggregators of each committee chosen by their real selection proofs
(up to TARGET_AGGREGATORS_PER_COMMITTEE = 16 per committee) and a planted share of exact duplicates, subsets and aggregates with a bad
signature.  Every signature is made with Engine.sign over messages tests/aggregate_intake_oracle.py computes.

    python tools/aggregate_intake_bench.py [--calls 5] [--rounds 3] [--share 0.05]
    python tools/aggregate_intake_bench.py --profile     # one torch.profiler pass: the split over the call's kernels

Reported:
  intake_ms          device time of Engine.aggregate_and_proof_intake_dev (CUDA events around --calls back-to-back calls, median and range
                     over the rounds);
  host_batched_ms    the three signature checks of the same items through the existing synchronous batched calls (Engine.fast_aggregate_verify
                     over the items' member rows and Engine.aggregate_verify over the 2n single-key sets), wall clock, the roots given;
  statuses           how many items ended with each status: the planted ones must read 10 (duplicates, subsets) and 16 (bad aggregates),
                     every other item 0.
Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import hashlib
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
from epoch_discount_bench import _card  # noqa: E402
from epoch_intake_bench import _tree_slots  # noqa: E402

DOMAINS = bytes([1] * 32) + bytes([5] * 32) + bytes([6] * 32)
R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def _sk8(values):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in values), dtype=np.uint32).reshape(-1, 8)


def _items(eng, W, slot, epoch, share):
    """wire records, woff, the planted kind per item (0 honest, 1 duplicate, 2 subset, 3 bad aggregate), and the verify inputs"""
    import aggregate_intake_oracle as A
    import intake_oracle as IO
    parent, roots, _ = W["tree"]
    K, C = bench.N_AGG, bench.COMMITTEE_SIZE
    spe, cps = bench.SLOTS, bench.COMMITTEES_PER_SLOT
    start = epoch * spe
    sk = lambda i: W["sk0"] + int(i) * W["delta"]      # noqa: E731
    members = W["members"]
    rng = np.random.default_rng(5)
    # selection proofs of every validator for its committee's slot, then is_aggregator
    com_of = np.repeat(np.arange(K), C)
    slot_msgs = np.frombuffer(b"".join(A.slot_signing_root(start + s, DOMAINS[32:64]) for s in range(spe)), np.uint8).reshape(spe, 32)
    proofs = eng.sign(_sk8([sk(v) for v in members]), (com_of // cps).astype(np.uint32), slot_msgs)
    modulo = max(1, C // 16)
    sel = np.array([int.from_bytes(hashlib.sha256(p.tobytes()).digest()[:8], "little") % modulo == 0 for p in proofs])
    datas, msgs = [], []
    for k in range(K):
        s = start + k // cps
        near = np.nonzero((slot <= s) & (slot + 4 > s))[0]
        h = int(near[k % len(near)])
        t = IO.ancestor(parent, slot, h, start)
        d = IO.data128(s, k % cps, bytes(roots[h]), epoch - 1, bytes(roots[0]), epoch, bytes(roots[t]))
        datas.append(d)
        msgs.append(A.signing_root(A.data_root(d), DOMAINS[0:32]))
    spec = []            # (committee, aggregator position, bits, kind)
    for k in range(K):
        pos = np.flatnonzero(sel[k * C:(k + 1) * C])[:16]
        for p in pos:
            r = rng.random()
            if spec and spec[-1][3] == 0 and r < share:
                spec.append(spec[-1][:3] + (1,))                                           # an exact duplicate of the previous item
            elif r < 2 * share:
                bits = rng.random(C) < 0.98
                spec.append((k, int(p), bits, 0))
                spec.append((k, int(pos[0]), bits & (rng.random(C) < 0.5), 2))             # a subset of it after it
            elif r < 3 * share:
                spec.append((k, int(p), rng.random(C) < 0.98, 3))
            else:
                spec.append((k, int(p), rng.random(C) < 0.98, 0))
    n = len(spec)
    # aggregate signatures: sk_i = sk0 + i * delta, so the selected members' key sum is count * sk0 + delta * (sum of their indices)
    agg_sk, agg_msg = [], []
    for k, p, bits, kind in spec:
        idx = members[k * C:(k + 1) * C][bits].astype(np.int64)
        agg_sk.append((len(idx) * W["sk0"] + W["delta"] * int(idx.sum())) % R_ORDER or 1)
        agg_msg.append(bytes(32) if kind == 3 else msgs[k])
    agg_sig = eng.sign(_sk8(agg_sk), np.arange(n, dtype=np.uint32), np.frombuffer(b"".join(agg_msg), np.uint8).reshape(n, 32))
    aap = []
    for i, (k, p, bits, kind) in enumerate(spec):
        v = int(members[k * C + p])
        aap.append(A.aggregate_and_proof_signing_root(v, bits.tolist(), datas[k], agg_sig[i].tobytes(), proofs[k * C + p].tobytes(), DOMAINS[64:96]))
    aggs = [int(members[k * C + p]) for k, p, _, _ in spec]
    outer = eng.sign(_sk8([sk(v) for v in aggs]), np.arange(n, dtype=np.uint32), np.frombuffer(b"".join(aap), np.uint8).reshape(n, 32))
    wires = [A.encode(aggs[i], spec[i][2].tolist(), datas[spec[i][0]], agg_sig[i].tobytes(), proofs[spec[i][0] * C + spec[i][1]].tobytes(),
                      outer[i].tobytes()) for i in range(n)]
    woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
    kinds = np.array([x[3] for x in spec])
    # the inputs of the existing batched calls: member rows, bit rows, messages; the single-key sets (proof, then outer signature)
    rows = np.zeros((n, C // 8), np.uint8)
    for i, (_, _, bits, _) in enumerate(spec):
        rows[i] = np.packbits(bits, bitorder="little")
    verify = dict(members=np.concatenate([members[k * C:(k + 1) * C] for k, _, _, _ in spec]), off=(np.arange(n + 1) * C).astype(np.uint32),
                  bits=rows, msgs=np.frombuffer(b"".join(msgs[k] for k, _, _, _ in spec), np.uint8).reshape(n, 32), agg_sig=agg_sig,
                  signers=np.repeat(np.array(aggs, np.uint32), 2),
                  sk_msgs=np.frombuffer(b"".join(slot_msgs[k // cps].tobytes() + aap[i] for i, (k, _, _, _) in enumerate(spec)), np.uint8).reshape(2 * n, 32),
                  sk_sigs=np.stack([np.stack([proofs[k * C + p], outer[i]]) for i, (k, p, _, _) in enumerate(spec)]).reshape(2 * n, 96))
    return b"".join(wires), woff, kinds, verify


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--share", type=float, default=0.05, help="share of items planted as each of: duplicate, subset, bad aggregate")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    assert torch.cuda.is_available(), "needs an H100: there is no CPU form of this measurement"
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    K, C = bench.N_AGG, bench.COMMITTEE_SIZE
    spe, cps = bench.SLOTS, bench.COMMITTEES_PER_SLOT
    parent, roots, leaf_viable = W["tree"]
    slot = _tree_slots(parent)
    eng.tree_load(parent, slot, roots, leaf_viable)
    epoch = int(slot.max()) // spe - 1
    current_slot = epoch * spe + spe - 1                  # the epoch's last slot: every item is inside the propagation range
    t0 = time.perf_counter()
    wire, woff, kinds, V = _items(eng, W, slot, epoch, a.share)
    setup_s = time.perf_counter() - t0
    n = len(woff) - 1
    t = lambda x: torch.as_tensor(np.array(x, copy=True)).to(dev)      # noqa: E731
    d_wire, d_woff = t(np.frombuffer(wire, np.uint8)), t(woff.view(np.int32))
    d_members, d_off = t(W["members"].astype(np.uint32).view(np.int32)), t(W["off"].astype(np.uint32).view(np.int32))
    z = lambda *s, dt=torch.int32: torch.zeros(s, dtype=dt, device=dev)      # noqa: E731
    outs = [z(n), z(n), z(n), z(n, C // 8, dt=torch.uint8), z(n, 96, dt=torch.uint8), z(n, 32, dt=torch.uint8), z(n, dt=torch.int64), z(n),
            z(n, C), z(n + 1)]

    def call(k):
        for _ in range(k):
            eng.aggregate_and_proof_intake_dev(d_wire, d_woff, d_members, d_off, epoch, current_slot, DOMAINS, cps, spe, *outs)

    call(2)
    torch.cuda.synchronize()
    status = outs[0].cpu().numpy()
    want = np.where(kinds == 0, 0, np.where(kinds == 3, 16, 10))
    assert np.array_equal(status, want), {int(s): int((status == s).sum()) for s in np.unique(status)}
    result = {"validators": bench.N_VAL, "committees": K, "committee_size": C, "items": n, "planted_share": a.share, "setup_s": round(setup_s, 1),
              "statuses": {str(int(s)): int((status == s).sum()) for s in np.unique(status)}}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(a.calls)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if total_us > 0:
                split[ev.key.split("(")[0][:60]] = round(total_us / 1e3 / a.calls, 4)
        result["device_ms_per_call"] = dict(sorted(split.items(), key=lambda kv: -kv[1]))
    else:
        ms, host = [], []
        for _ in range(a.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            call(a.calls)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / a.calls)
            h0 = time.perf_counter()
            ok_fav = eng.fast_aggregate_verify(V["members"], V["off"], V["bits"], V["msgs"], V["agg_sig"])
            ok_av = eng.aggregate_verify(V["signers"], np.arange(2 * n + 1, dtype=np.uint32), V["sk_msgs"], V["sk_sigs"])
            host.append((time.perf_counter() - h0) * 1e3)
            assert np.array_equal(ok_fav.astype(bool), kinds != 3) and bool(ok_av.all())
        result.update({"intake_ms": round(float(np.median(ms)), 3), "intake_ms_range": [round(min(ms), 3), round(max(ms), 3)],
                       "host_batched_ms": round(float(np.median(host)), 3), "host_batched_ms_range": [round(min(host), 3), round(max(host), 3)],
                       "calls_per_round": a.calls, "rounds": a.rounds})
    assert eng.guard_flags() == 0
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
