"""What slashing detection costs the epoch pipeline: bench.py's epoch (2^20 validators, 2 048 committees x 512, depth 3, inputs built by
bench.build_world) through EpochProcessor.submit_dev with and without enable_slasher, alternating in one process on one Engine.

    python tools/epoch_slasher_bench.py [--history 4096] [--epochs 60] [--rounds 3] [--planted 4] [--depth 3]
    python tools/epoch_slasher_bench.py --profile [--epochs 8]          # one torch.profiler pass: device time per kernel under the pipeline

The ring starts at --history epochs and is halved until b2_slasher_init stops refusing with B2_ENOMEM (the size used is printed); it
is allocated after both processors have run, so the refusal is against the memory the pipeline leaves.  Offences are planted through
the pipeline's own inputs (the committees are fixed, so aggregate a has the same members every epoch): in epoch k, --planted
aggregates carry target k-1 and another message, signed with the members' keys by bls.Sign on the GPU (double votes of every member),
and --planted others carry source k-3 (they surround the members' (k-2, k-1) vote); which aggregates alternates with the parity of k.
Every epoch's flagged count must equal committee size x planted aggregates (after the slasher's first epoch, which has no history).
Per round: `epochs` epochs without the slasher, then the same epochs with it; CUDA events around each batch (fill and drain included,
every ticket waited for, the slasher's count read per epoch); median and range over the rounds.  Then an untimed pass checks that
verdicts, heads and aggregate signatures are byte-identical with the slasher on and off.  Prints one JSON line with the card's name
and power limit, read in the same run.  Writes nothing."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402


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


class Inputs:
    """the two input variants (by the parity of k) and the per-epoch source / target epochs, all on the device"""

    def __init__(self, eng, W, planted, dev):
        import torch
        self.torch = torch
        A, C = bench.N_AGG, bench.COMMITTEE_SIZE
        step = A // (4 * planted)
        self.double = [[(4 * i + 2 * p) * step for i in range(planted)] for p in (0, 1)]
        self.surround = [[(4 * i + 2 * p + 1) * step for i in range(planted)] for p in (0, 1)]
        self.d_sigs, self.d_msgs, self.d_tgt_pat, self.d_src_pat = [], [], [], []
        for p in (0, 1):
            sigs, msgs = W["sigs"].copy(), W["msgs"].copy()
            tgt, src = np.zeros(A, dtype=np.int64), np.full(A, -1, dtype=np.int64)
            for a in self.double[p]:
                msgs[a] = np.frombuffer(hashlib.sha256(b"other/%d" % a).digest(), dtype=np.uint8)
                m = W["members"][a * C:(a + 1) * C]
                sks = [(W["sk0"] + int(v) * W["delta"]) % bench.R_ORDER for v in m]
                sigs[a * C:(a + 1) * C] = eng.sign(sks, np.zeros(C, dtype=np.uint32), msgs[a:a + 1])
                tgt[a], src[a] = -1, -2
            for a in self.surround[p]:
                src[a] = -3
            self.d_sigs.append(torch.as_tensor(sigs, device=dev))
            self.d_msgs.append(torch.as_tensor(msgs, device=dev))
            self.d_tgt_pat.append(torch.as_tensor(tgt, device=dev))
            self.d_src_pat.append(torch.as_tensor(src, device=dev))
        self.d_bits = torch.full((A, C // 8), 0xFF, dtype=torch.uint8, device=dev)
        self.d_blk = torch.as_tensor((bench.N_BLOCKS - 1 - (np.arange(A) % 64)).astype(np.int32), device=dev)
        self.d_tgt = torch.zeros(A, dtype=torch.int64, device=dev)
        self.d_src = torch.zeros(A, dtype=torch.int64, device=dev)
        self.planted_slots = 2 * planted * C

    def args(self, k):
        """epoch k's arguments, prepared on the current stream (submit_dev copies the epochs into the slot in stream order)"""
        p = k & 1
        self.torch.add(self.d_tgt_pat[p], k, out=self.d_tgt)
        self.torch.add(self.d_src_pat[p], k, out=self.d_src)
        return (self.d_sigs[p], self.d_bits, self.d_msgs[p], self.d_tgt, self.d_blk), self.d_src


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--history", type=int, default=4096)
    ap.add_argument("--epochs", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--planted", type=int, default=4, help="aggregates per epoch with a double vote, and as many with a surround vote")
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200._lib import B2_ENOMEM, B2Error
    from pos_evolution_b200.engine import Engine
    from pos_evolution_b200.epoch import EpochProcessor
    assert torch.cuda.is_available(), "needs an H100: there is no CPU form of this measurement"
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    W = bench.build_world(eng, 0, np, PS)
    inp = Inputs(eng, W, a.planted, dev)
    boost = (bench.N_BLOCKS - 1, W["boost"])
    procs = {}
    for name in ("off", "on"):
        ep = EpochProcessor(eng, bench.N_AGG, bench.N_VAL, bench.COMMITTEE_SIZE // 8, bench.N_BLOCKS, device=dev, depth=a.depth)
        ep.set_committees(W["members"], W["off"])
        procs[name] = ep
    state = {"k": 1000}                      # the slasher's epochs; the runs without it replay the same k

    def run(name, ks, collect=False):
        ep, out = procs[name], []
        for i, k in enumerate(ks):
            args, src = inp.args(k)
            kw = dict(source_epoch=src, current_epoch=k) if ep.slasher else {}
            t = ep.submit_dev(*args, 0, boost[0], boost[1], last=ep.drain_hint(len(ks) - 1 - i), **kw)
            if t is not None:
                out.append(t)
                _take(t, ep, collect)
        for t in ep.drain():
            out.append(t)
            _take(t, ep, collect)
        return out

    def _take(t, ep, collect):
        ok, head = t.wait()
        t.flagged = t.n_flagged() if ep.slasher else None
        if collect:
            t.digest = hashlib.sha256(ok.cpu().numpy().tobytes() + int(head).to_bytes(4, "little") +
                                      t.aggregate_signatures().cpu().numpy().tobytes()).hexdigest()

    # warm-up of both processors (the library's scratch is allocated), then the slasher, as large as the card allows
    for name in ("off", "on"):
        run(name, range(990, 990 + a.depth + 1))
    torch.cuda.synchronize()
    H = a.history
    while True:
        try:
            procs["on"].enable_slasher(H, current_epoch=state["k"])
            break
        except B2Error as e:
            if e.code != B2_ENOMEM or H <= 64:
                raise
            H //= 2
    K = min(2 * bench.N_AGG, 65535)
    result = {"validators": bench.N_VAL, "aggregates_per_epoch": bench.N_AGG, "committee_size": bench.COMMITTEE_SIZE, "depth": a.depth,
              "history_epochs": H, "history_epochs_asked": a.history, "max_attestations_per_target": K,
              "slasher_bytes": 6 * bench.N_VAL * H + 32 * H * K + 4 * H, "planted_aggregates_per_epoch": 2 * a.planted,
              "planted_slots_per_epoch": inp.planted_slots}

    def next_ks(n):
        ks = list(range(state["k"], state["k"] + n))
        state["k"] += n
        return ks

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        run("on", next_ks(a.depth + 2))
        torch.cuda.synchronize()
        ks = next_ks(a.epochs)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run("on", ks)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if total_us > 0:
                split[ev.key.split("(")[0][:60]] = round(total_us / 1e3 / len(ks), 4)
        result["profile_epochs"] = len(ks)
        result["device_ms_per_epoch_by_kernel"] = dict(sorted(split.items(), key=lambda kv: -kv[1])[:25])
        result["slasher_ms_per_epoch"] = round(sum(v for k, v in split.items() if "k_slasher" in k), 4)
    else:
        ms = {"off": [], "on": []}
        first = True
        for _ in range(a.rounds):
            ks = next_ks(a.epochs)
            for name in ("off", "on"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                tickets = run(name, ks)
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1) / len(ks))
                if name == "on":
                    flagged = [t.flagged for t in tickets]
                    want = [0 if (first and i == 0) else inp.planted_slots for i in range(len(ks))]
                    assert flagged == want, ("flagged", flagged, "planted", want)
                    first = False
        ks = next_ks(2 * a.depth + 2)
        dig = {name: [t.digest for t in run(name, ks, collect=True)] for name in ("off", "on")}
        assert dig["off"] == dig["on"], "verdicts, heads or aggregate signatures differ with the slasher on"
        assert eng.guard_flags() == 0
        med = {n: float(np.median(v)) for n, v in ms.items()}
        result.update({"epochs_per_round": a.epochs, "rounds": a.rounds,
                       "ms_per_epoch_off": round(med["off"], 3), "ms_per_epoch_on": round(med["on"], 3),
                       "ms_per_epoch_off_range": [round(min(ms["off"]), 3), round(max(ms["off"]), 3)],
                       "ms_per_epoch_on_range": [round(min(ms["on"]), 3), round(max(ms["on"]), 3)],
                       "overhead_pct": round(100.0 * (med["on"] / med["off"] - 1.0), 2),
                       "flagged_equals_planted": True, "outputs_identical_on_off": True})
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
