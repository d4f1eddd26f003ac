"""What equivocation discounting costs the epoch pipeline: bench.py's epoch (2^20 validators, 2 048 committees x 512, depth 3, inputs built
by bench.build_world) through EpochProcessor.submit_dev with the slasher on and planted offences (those of tools/epoch_slasher_bench.py),
with enable_slasher(..., discount=False) and discount=True, alternating in one process on one Engine.

    python tools/epoch_discount_bench.py [--history 1024] [--epochs 60] [--rounds 3] [--planted 4] [--depth 3]
    python tools/epoch_discount_bench.py --profile [--epochs 8]         # one torch.profiler pass: device time per kernel under the pipeline

The two processors share the Engine's one slasher (its ring starts at --history epochs and is halved until b2_slasher_init stops
refusing with B2_ENOMEM), fed increasing epochs in turn.  Every batch starts from an empty equivocating table (latest_messages_reset,
outside the timed window), so with discounting on the first two epochs of a batch each newly mark the 2 x planted x 512 validators of
one parity's offences and every later epoch marks none; that count is checked per epoch.  CUDA events around each batch (fill and
drain included, every ticket waited for); median and range over the rounds.  Then an untimed pass checks every epoch's discounted
validators against the host oracle (the slasher's flagged validators not yet equivocating).  Heads are not compared: discounting
changes them by design.  Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
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
    ap.add_argument("--history", type=int, default=1024)
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
    state = {"k": 1000}

    def run(name, ks, collect=False):
        ep, out = procs[name], []
        for i, k in enumerate(ks):
            args, src = inp.args(k)
            t = ep.submit_dev(*args, 0, boost[0], boost[1], last=ep.drain_hint(len(ks) - 1 - i), source_epoch=src, current_epoch=k)
            if t is not None:
                out.append(t)
                _take(t, ep, collect)
        for t in ep.drain():
            out.append(t)
            _take(t, ep, collect)
        return out

    def _take(t, ep, collect):
        t.wait()
        t.new = t.discounted() if ep.discount else None
        if collect:
            t.flagged_validators = np.unique(t.slashings().validator)

    # the slasher, as large as the card allows; the "off" processor's enable_slasher is replaced by the "on" one's init, and both then
    # feed the same history with increasing epochs
    H = a.history
    while True:
        try:
            eng.slasher_free()
            procs["off"].enable_slasher(H, current_epoch=state["k"], discount=False)
            procs["on"].enable_slasher(H, current_epoch=state["k"], discount=True)
            break
        except B2Error as e:
            if e.code != B2_ENOMEM or H <= 64:
                raise
            H //= 2
    K = min(2 * bench.N_AGG, 65535)
    result = {"validators": bench.N_VAL, "aggregates_per_epoch": bench.N_AGG, "committee_size": bench.COMMITTEE_SIZE, "depth": a.depth,
              "history_epochs": H, "max_attestations_per_target": K, "planted_aggregates_per_epoch": 2 * a.planted,
              "planted_slots_per_epoch": inp.planted_slots}

    def next_ks(n):
        ks = list(range(state["k"], state["k"] + n))
        state["k"] += n
        return ks

    # warm-up of both processors (the library's scratch is allocated, the slasher gets a history)
    for name in ("off", "on"):
        run(name, next_ks(a.depth + 2))
    torch.cuda.synchronize()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        eng.latest_messages_reset()
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
        result["discount_ms_per_epoch"] = round(sum(v for k, v in split.items() if "k_slasher_discount" in k), 5)
        result["slasher_ms_per_epoch"] = round(sum(v for k, v in split.items() if "k_slasher" in k), 4)
    else:
        ms = {"off": [], "on": []}
        for _ in range(a.rounds):
            for name in ("off", "on"):
                ks = next_ks(a.epochs)
                eng.latest_messages_reset()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                tickets = run(name, ks)
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1) / len(ks))
                if name == "on":
                    got = [len(t.new) for t in tickets]
                    want = [inp.planted_slots if i < 2 else 0 for i in range(len(ks))]
                    assert got == want, ("newly discounted", got, "expected", want)
        # untimed: every epoch's discounted validators against the host oracle
        eng.latest_messages_reset()
        E = set()
        for t in run("on", next_ks(2 * a.depth + 2), collect=True):
            want = sorted(set(t.flagged_validators.tolist()) - E)
            assert t.new.tolist() == want, "discounted validators differ from the oracle"
            E |= set(want)
        assert len(E) == 2 * inp.planted_slots and int((procs["on"].equivocating() != 0).sum()) == len(E)
        assert eng.guard_flags() == 0
        med = {n: float(np.median(v)) for n, v in ms.items()}
        result.update({"epochs_per_round": a.epochs, "rounds": a.rounds,
                       "ms_per_epoch_off": round(med["off"], 3), "ms_per_epoch_on": round(med["on"], 3),
                       "ms_per_epoch_off_range": [round(min(ms["off"]), 3), round(max(ms["off"]), 3)],
                       "ms_per_epoch_on_range": [round(min(ms["on"]), 3), round(max(ms["on"]), 3)],
                       "overhead_pct": round(100.0 * (med["on"] / med["off"] - 1.0), 2),
                       "discounted_equals_oracle": True})
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
