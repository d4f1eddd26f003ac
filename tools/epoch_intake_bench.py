"""What the attestation intake costs: bench.py's epoch (2^20 validators, 2 048 committees x 512, depth 3, keys and committees from
bench.build_world) arriving as 2^20 unaggregated Attestations on the wire, in random order, with 1, 2 and 4 votes per committee (each
vote a different head of the 10 000-block tree, each member signing its vote's real signing root with Engine.sign).

    python tools/epoch_intake_bench.py [--epochs 20] [--rounds 3] [--depth 3]
    python tools/epoch_intake_bench.py --profile         # one torch.profiler pass per case: the split over the intake's kernels
    python tools/epoch_intake_bench.py --form electra    # the same epochs also as Electra SingleAttestations, beside the phase 0 form

Reported per case:
  intake_ms            device time of Engine.attestation_intake_dev (CUDA events around --epochs back-to-back calls, median and range
                       over the rounds);
  ms_per_epoch_*       a pipelined epoch (EpochProcessor.submit_dev in the vote form) fed by EpochProcessor.intake_dev on a side stream
                       each epoch ("intake"), against the same epoch fed the votes one intake produced beforehand ("precomputed"),
                       alternating in one process (CUDA events around each batch, fill and drain included);
  host_numpy_ms        the numpy oracle (tests/intake_oracle.intake_numpy) computing the same outputs on this host's CPU (one run).
With --form electra every case also holds the same votes as 2^20 SingleAttestations (data.index = 0, signed as such, on their committees'
subnets), and adds single_intake_ms (Engine.single_attestation_intake_dev, as intake_ms) and ms_per_epoch_single_intake (the pipelined
epoch fed by EpochProcessor.intake_single_dev), alternating with the phase 0 rows; --profile then splits both calls.
Every kept attestation must be status 0 and every vote must verify.  Prints one JSON line with the card's name and power limit, read in
the same run.  Writes nothing."""
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
from epoch_discount_bench import _card  # noqa: E402
from epoch_votes_bench import _secret_keys  # noqa: E402

CASES = (1, 2, 4)
DOMAIN = bytes(range(32))


def _tree_slots(parent):
    """one slot per block, one more than its parent's: strictly increasing along every chain"""
    slot = np.zeros(parent.shape[0], dtype=np.uint64)
    for b in range(1, parent.shape[0]):
        slot[b] = slot[parent[b]] + 1
    return slot


def _epoch(eng, W, slot, n_votes_per, epoch, electra=False):
    """uint8[n, L] wire records of one epoch in random order and its vote count; electra: 240-byte SingleAttestations of data with
    data.index = 0, and the subnet of each record"""
    import intake_oracle as IO
    parent, roots, _ = W["tree"]
    A, C = bench.N_AGG, bench.COMMITTEE_SIZE
    spe, cps = bench.SLOTS, bench.COMMITTEES_PER_SLOT
    start = epoch * spe
    rng = np.random.default_rng(7 * n_votes_per)
    data = np.zeros((A, n_votes_per, 128), dtype=np.uint8)
    for k in range(A):
        s = start + k // cps
        near = np.nonzero((slot <= s) & (slot + 4 > s))[0]
        for v in range(n_votes_per):
            h = int(near[(k + 17 * v) % len(near)])
            t = IO.ancestor(parent, slot, h, start)
            data[k, v] = np.frombuffer(IO.data128(s, 0 if electra else k % cps, bytes(roots[h]), epoch - 1, bytes(roots[0]), epoch,
                                                  bytes(roots[t])), np.uint8)
    msgs = eng.signing_roots(data.reshape(-1, 128), np.frombuffer(DOMAIN, np.uint8))
    com = np.repeat(np.arange(A, dtype=np.int64), C)
    pos = np.tile(np.arange(C), A)
    vote = com * n_votes_per + rng.integers(0, n_votes_per, size=A * C)
    sigs = eng.sign(_secret_keys(W)[W["members"]], vote.astype(np.uint32), msgs)
    if electra:                       # committee k's members are W["members"][k * C .. (k + 1) * C)
        rec = np.zeros((A * C, 240), dtype=np.uint8)
        rec[:, 0:8] = (com % cps).astype("<u8").view(np.uint8).reshape(-1, 8)
        rec[:, 8:16] = W["members"].astype("<u8").view(np.uint8).reshape(-1, 8)
        rec[:, 16:144] = data.reshape(-1, 128)[vote]
        rec[:, 144:240] = sigs
        order = rng.permutation(A * C)
        return rec[order], A * n_votes_per, (com % 64).astype(np.uint32)[order]      # compute_subnet_for_attestation = k % 64 here
    L = 228 + C // 8 + 1
    rec = np.zeros((A * C, L), dtype=np.uint8)
    rec[:, 0] = 228
    rec[:, 4:132] = data.reshape(-1, 128)[vote]
    rec[:, 132:228] = sigs
    rec[np.arange(A * C), 228 + pos // 8] = (1 << (pos % 8)).astype(np.uint8)
    rec[:, L - 1] |= 1
    return rec[rng.permutation(A * C)], A * n_votes_per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--form", choices=("phase0", "electra"), default="phase0")
    a = ap.parse_args()
    import torch
    import intake_oracle as IO
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    assert torch.cuda.is_available(), "needs an H100: there is no CPU form of this measurement"
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    A, C = bench.N_AGG, bench.COMMITTEE_SIZE
    spe, cps = bench.SLOTS, bench.COMMITTEES_PER_SLOT
    parent, roots, leaf_viable = W["tree"]
    slot = _tree_slots(parent)
    eng.tree_load(parent, slot, roots, leaf_viable)
    epoch = int(slot.max()) // spe - 1
    current_slot = (epoch + 1) * spe + 1
    ep = EpochProcessor(eng, A, bench.N_VAL, C // 8, bench.N_BLOCKS, device=dev, depth=a.depth, max_votes=A * max(CASES))
    ep.set_committees(W["members"], W["off"])
    side = torch.cuda.Stream()
    electra = a.form == "electra"
    assert not electra or np.array_equal(W["off"], np.arange(A + 1) * C)
    result = {"validators": bench.N_VAL, "committees": A, "committee_size": C, "depth": a.depth, "attestations": A * C, "form": a.form}
    rows = {}
    for n_votes_per in CASES:
        rec, n_votes = _epoch(eng, W, slot, n_votes_per, epoch)
        L = rec.shape[1]
        d_wire = torch.as_tensor(rec.reshape(-1), device=dev)
        d_woff = torch.as_tensor((np.arange(rec.shape[0] + 1, dtype=np.int64) * L).astype(np.int32), device=dev)
        args = (d_wire, d_woff, epoch, current_slot, DOMAIN, cps, spe)
        with torch.cuda.stream(side):
            pre = ep.intake_dev(*args)
        assert bool((pre.status == 0).all()) and int(pre.vote_off[-1]) == n_votes
        if electra:
            rec1, _, sub1 = _epoch(eng, W, slot, n_votes_per, epoch, electra=True)
            d_wire1 = torch.as_tensor(rec1.reshape(-1), device=dev)
            d_woff1 = torch.as_tensor((np.arange(rec1.shape[0] + 1, dtype=np.int64) * 240).astype(np.int32), device=dev)
            d_sub1 = torch.as_tensor(sub1.view(np.int32), device=dev)
            args1 = (d_wire1, d_woff1, d_sub1, epoch, current_slot, DOMAIN, cps, spe)
            with torch.cuda.stream(side):
                pre1 = ep.intake_single_dev(*args1)
            assert bool((pre1.status == 0).all()) and np.array_equal(pre1.vote_off, pre.vote_off)
            assert torch.equal(pre1.vote, pre.vote)         # the same votes (the signatures differ: data.index is 0 in what they sign)

        def pipelined(n, fresh):
            out, inputs = [], []          # every epoch's intake stays alive until its ticket has been waited for
            for i in range(n):
                if fresh == "single":
                    with torch.cuda.stream(side):
                        r = ep.intake_single_dev(*args1)
                elif fresh:
                    with torch.cuda.stream(side):
                        r = ep.intake_dev(*args)
                else:
                    r = pre
                inputs.append(r)
                t = ep.submit_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, last=ep.drain_hint(n - 1 - i), votes=(r.vote, r.vote_off))
                out += [t] if t is not None else []
            out += ep.drain()
            return [t.wait()[0] for t in out]

        # the intake alone, on preallocated outputs
        z = lambda *s, dt=torch.uint8: torch.zeros(s, dtype=dt, device=dev)      # noqa: E731
        mv = ep.max_votes
        outs = [z(rec.shape[0], dt=torch.int32), z(A * C, dt=torch.int32), z(A + 1, dt=torch.int32), z(A * C, 96), z(mv, 128), z(mv, 32),
                z(mv, dt=torch.int64), z(mv, dt=torch.int64), z(mv, dt=torch.int32)]

        def intake_only(n):
            for _ in range(n):
                eng.attestation_intake_dev(d_wire, d_woff, ep.d_off, epoch, current_slot, DOMAIN, cps, spe, C // 8, *outs)

        def single_intake_only(n):
            for _ in range(n):
                eng.single_attestation_intake_dev(d_wire1, d_woff1, d_sub1, ep.d_members, ep.d_off, epoch, current_slot, DOMAIN, cps, spe,
                                                  C // 8, *outs)

        feeds = (True, False, "single") if electra else (True, False)
        for fresh in feeds:                               # warm-up: every shape of the timed window
            assert all(bool(x.all()) for x in pipelined(a.depth + 2, fresh)), "every vote of the warm-up must verify"
        intake_only(3)
        if electra:
            single_intake_only(3)
        torch.cuda.synchronize()
        row = {"n_votes": n_votes}
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            for name, fn in [("device_ms_per_intake", intake_only)] + ([("device_ms_per_single_intake", single_intake_only)] if electra else []):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn(a.epochs)
                    torch.cuda.synchronize()
                split = {}
                for ev in prof.key_averages():
                    total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    if total_us > 0 and ("k_intake" in ev.key or "k_single" in ev.key or "Memset" in ev.key):
                        split[ev.key.split("(")[0][:60]] = round(total_us / 1e3 / a.epochs, 4)
                row[name] = split
        else:
            names = ("intake", "precomputed", "intake_only") + (("single_intake", "single_intake_only") if electra else ())
            ms = {name: [] for name in names}
            for _ in range(a.rounds):
                for name in names:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    if name == "intake_only":
                        intake_only(a.epochs)
                    elif name == "single_intake_only":
                        single_intake_only(a.epochs)
                    else:
                        ok = pipelined(a.epochs, "single" if name == "single_intake" else name == "intake")
                    e1.record()
                    torch.cuda.synchronize()
                    ms[name].append(e0.elapsed_time(e1) / a.epochs)
                    if not name.endswith("intake_only"):
                        assert all(bool(x.all()) for x in ok), (name, n_votes_per, "every vote must verify")
            med = {k: float(np.median(v)) for k, v in ms.items()}
            t0 = time.perf_counter()
            ref = IO.intake_numpy(rec, W["off"].astype(np.int64), epoch, current_slot, DOMAIN, cps, spe, C // 8, parent, slot, roots)
            host_ms = (time.perf_counter() - t0) * 1e3
            assert np.array_equal(ref.vote_off, pre.vote_off) and np.array_equal(ref.msgs[:n_votes], pre.msgs[:n_votes].cpu().numpy())
            row.update({"intake_ms": round(med["intake_only"], 3), "intake_ms_range": [round(min(ms["intake_only"]), 3), round(max(ms["intake_only"]), 3)],
                        "ms_per_epoch_intake": round(med["intake"], 3), "ms_per_epoch_precomputed": round(med["precomputed"], 3),
                        "ms_range_intake": [round(min(ms["intake"]), 3), round(max(ms["intake"]), 3)],
                        "ms_range_precomputed": [round(min(ms["precomputed"]), 3), round(max(ms["precomputed"]), 3)],
                        "host_numpy_ms": round(host_ms, 1)})
            if electra:
                row.update({"single_intake_ms": round(med["single_intake_only"], 3),
                            "single_intake_ms_range": [round(min(ms["single_intake_only"]), 3), round(max(ms["single_intake_only"]), 3)],
                            "ms_per_epoch_single_intake": round(med["single_intake"], 3),
                            "ms_range_single_intake": [round(min(ms["single_intake"]), 3), round(max(ms["single_intake"]), 3)]})
        rows["%dv" % n_votes_per] = row
        del d_wire, pre
        if electra:
            del d_wire1, pre1
    result.update({"epochs_per_round": a.epochs, "rounds": a.rounds, "cases": rows, "host_cpu": os.cpu_count()})
    assert eng.guard_flags() == 0
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
