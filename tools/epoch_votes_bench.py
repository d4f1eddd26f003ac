"""What the vote form of the epoch pipeline costs: bench.py's epoch (2^20 validators, 2 048 committees x 512, depth 3, inputs built by
bench.build_world) through EpochProcessor.submit_dev in the committee form and in the vote form (votes=(vote, vote_off)), alternating in
one process on one Engine, at

    1 vote per committee, 100 % participation   the cost of the grouping alone (the grouped arrays equal the inputs)
    2 and 4 votes per committee, 100 %          each member signs its vote's message (Engine.sign with a per-member message index)
    2 votes per committee, 95 %                 non-attesters: their slots become the infinity encoding on the device

    python tools/epoch_votes_bench.py [--epochs 30] [--rounds 3] [--depth 3]
    python tools/epoch_votes_bench.py --profile [--epochs 8]        # one torch.profiler pass per case: the grouping kernel's device time

A split epoch verifies n_votes aggregates instead of 2 048: its pairings (2 Miller loops + 1 final exponentiation per aggregate) grow with
n_votes and are reported as such.  Every vote of every case must verify.  CUDA events around each batch of --epochs epochs (fill and
drain included, every ticket waited for); median and range over the rounds.  The host alternative -- a numpy stable argsort of the
same vote ids by (committee, vote) plus the permutation of the signatures and members -- is timed on this host's CPU (one core).
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

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402
from epoch_discount_bench import _card  # noqa: E402

NONE = 0xFFFFFFFF
CASES = [(1, 1.0), (2, 1.0), (4, 1.0), (2, 0.95)]


def _secret_keys(W):
    """sk_i = sk0 + i * delta as 8 little-endian u32 limbs per validator (bench.build_world's keys)"""
    b = b"".join((W["sk0"] + i * W["delta"]).to_bytes(32, "little") for i in range(bench.N_VAL))
    return np.frombuffer(b, dtype=np.uint32).reshape(bench.N_VAL, 8)


def _vote_case(eng, W, n_votes_per, participation, dev):
    """device inputs of one case: signatures, per-vote messages / epochs / blocks, vote ids, vote_off"""
    import torch
    A, C = bench.N_AGG, bench.COMMITTEE_SIZE
    rng = np.random.default_rng(1000 * n_votes_per + int(100 * participation))
    com = np.repeat(np.arange(A, dtype=np.int64), C)
    if n_votes_per == 1:
        vote = com.copy()
        msgs, sigs = W["msgs"], W["sigs"]
    else:
        vote = com * n_votes_per + rng.integers(0, n_votes_per, size=A * C)
        msgs = np.frombuffer(b"".join(hashlib.sha256(b"vote/%d" % v).digest() for v in range(A * n_votes_per)), dtype=np.uint8).reshape(-1, 32)
        sigs = eng.sign(_secret_keys(W)[W["members"]], vote.astype(np.uint32), msgs)
    if participation < 1.0:
        vote = np.where(rng.random(A * C) < participation, vote, NONE)
    n_votes = A * n_votes_per
    vote_off = np.arange(A + 1, dtype=np.int64) * n_votes_per
    blk = (bench.N_BLOCKS - 1 - (np.arange(n_votes) % 64)).astype(np.int32)
    return dict(vote=vote.astype(np.uint32), vote_off=vote_off, n_votes=n_votes,
                d=(torch.as_tensor(sigs, device=dev), None, torch.as_tensor(msgs, device=dev), torch.full((n_votes,), 5, dtype=torch.int64, device=dev),
                   torch.as_tensor(blk, device=dev)),
                d_vote=torch.as_tensor(vote.astype(np.uint32).view(np.int32), device=dev))


def _host_grouping_ms(W, case, reps=3):
    """numpy: stable argsort of the vote ids by (committee, vote, non-attesters last), then the permutation of signatures and members"""
    A, C = bench.N_AGG, bench.COMMITTEE_SIZE
    vote, sigs, members = case["vote"].astype(np.int64), W["sigs"], W["members"]
    com = np.repeat(np.arange(A, dtype=np.int64), C)
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        key = np.where(vote == NONE, case["vote_off"][com + 1], vote)      # a non-attester sorts after its committee's last vote
        p = np.argsort(key, kind="stable")
        g_sigs, g_members = sigs[p], members[p]
        out.append((time.perf_counter() - t0) * 1e3)
        assert g_sigs.shape == sigs.shape and g_members.shape == members.shape
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    assert torch.cuda.is_available(), "needs an H100: there is no CPU form of this measurement"
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    A, C = bench.N_AGG, bench.COMMITTEE_SIZE
    boost = (bench.N_BLOCKS - 1, W["boost"])
    base = (torch.as_tensor(W["sigs"], device=dev), torch.full((A, C // 8), 0xFF, dtype=torch.uint8, device=dev), torch.as_tensor(W["msgs"], device=dev),
            torch.full((A,), 5, dtype=torch.int64, device=dev), torch.as_tensor((bench.N_BLOCKS - 1 - (np.arange(A) % 64)).astype(np.int32), device=dev))
    committee = EpochProcessor(eng, A, bench.N_VAL, C // 8, bench.N_BLOCKS, device=dev, depth=a.depth)
    committee.set_committees(W["members"], W["off"])
    votes = EpochProcessor(eng, A, bench.N_VAL, C // 8, bench.N_BLOCKS, device=dev, depth=a.depth, max_votes=A * max(v for v, _ in CASES))
    votes.set_committees(W["members"], W["off"])
    cases = {(v, p): _vote_case(eng, W, v, p, dev) for v, p in CASES}

    def run(case, n):
        ep = committee if case is None else votes
        out = []
        for i in range(n):
            kw = {} if case is None else {"votes": (case["d_vote"], case["vote_off"])}
            args = base if case is None else case["d"]
            t = ep.submit_dev(*args, 0, boost[0], boost[1], last=ep.drain_hint(n - 1 - i), **kw)
            out += [t] if t is not None else []
        out += ep.drain()
        return [t.wait()[0] for t in out]

    for case in [None] + list(cases.values()):            # warm-up: every shape of the timed window
        ok = run(case, a.depth + 2)
        assert all(bool(x.all()) for x in ok), "every aggregate of the warm-up must verify"
    torch.cuda.synchronize()
    result = {"validators": bench.N_VAL, "committees": A, "committee_size": C, "depth": a.depth}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        prof_out = {}
        for (v, p), case in cases.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(case, a.epochs)
                torch.cuda.synchronize()
            split = {}
            for ev in prof.key_averages():
                total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                if total_us > 0:
                    split[ev.key.split("(")[0][:60]] = total_us / 1e3 / a.epochs
            prof_out["%dv_%d%%" % (v, round(100 * p))] = {
                "k_votes_group_ms": round(sum(t for k, t in split.items() if "k_votes_group" in k), 4),
                "k_votes_empty_ms": round(sum(t for k, t in split.items() if "k_votes_empty" in k), 4)}
        result["device_ms_per_epoch"] = prof_out
        result["profile_epochs"] = a.epochs
    else:
        rows = {}
        for (v, p), case in cases.items():
            ms = {"committee": [], "votes": []}
            for _ in range(a.rounds):
                for name, c in (("committee", None), ("votes", case)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    ok = run(c, a.epochs)
                    e1.record()
                    torch.cuda.synchronize()
                    ms[name].append(e0.elapsed_time(e1) / a.epochs)
                    assert all(bool(x.all()) for x in ok), (name, v, p, "every aggregate must verify")
            med = {n: float(np.median(x)) for n, x in ms.items()}
            rows["%dv_%d%%" % (v, round(100 * p))] = {
                "n_votes": case["n_votes"], "pairings_per_epoch_committee": 2 * A, "pairings_per_epoch_votes": 2 * case["n_votes"],
                "ms_per_epoch_committee": round(med["committee"], 3), "ms_per_epoch_votes": round(med["votes"], 3),
                "ms_range_committee": [round(min(ms["committee"]), 3), round(max(ms["committee"]), 3)],
                "ms_range_votes": [round(min(ms["votes"]), 3), round(max(ms["votes"]), 3)],
                "overhead_pct": round(100.0 * (med["votes"] / med["committee"] - 1.0), 2),
                "host_numpy_grouping_ms": round(_host_grouping_ms(W, case), 2)}
        result.update({"epochs_per_round": a.epochs, "rounds": a.rounds, "cases": rows, "host_cpu": os.cpu_count()})
        assert eng.guard_flags() == 0
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
