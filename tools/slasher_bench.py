"""The slasher (b2_slasher_update_dev) at full size: 2^20 validators, a ring of 4 096 epochs (25.8 GB of span tables; halved until it
fits the free memory of the card, and the size used is printed), one epoch batch = 2 048 aggregates x 512 members cut from
b2_shuffle_committees, every validator attesting honestly (cur - 1, cur), plus a planted share of offenders (0 %, 0.1 %, 5 %) who sign a
second, conflicting attestation in further aggregates of the same batch: alternately another head for the same target (double vote)
and (cur - 3, cur), which also surrounds their vote of the epoch before.

    python tools/slasher_bench.py [--validators 1048576] [--history 4096] [--warmup 3] [--epochs 20] [--rounds 3]

Per offender share: `warmup` epochs, then `epochs` timed ones, CUDA events around each epoch's update (rows + record + check kernels);
median and range over `rounds` rounds; b2_slasher_advance (column reset, synchronises) is timed by the host clock beside it.  The
flagged count of every epoch must equal the number planted.  The split between the kernels comes from one torch.profiler pass over
five more epochs.  Algorithmic bytes are computed from the shapes (every table cell counted once per access, 2 bytes).  Prints one
JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_AGG, CSIZE, PER_TARGET = 2048, 512, 4096


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


class Stream:
    """epoch batches on the device; shuffles come from a small pool, offenders are a fresh sample each epoch"""

    def __init__(self, eng, n, share, seed):
        import torch
        self.torch, self.eng, self.n = torch, eng, n
        self.rng = np.random.default_rng(seed)
        self.n_extra = int(round(share * n / CSIZE))
        self.n_agg = n // CSIZE + self.n_extra
        self.total = self.n_agg * CSIZE
        dev = torch.device("cuda", 0)
        self.pool = [torch.as_tensor(eng.shuffle_committees(bytes([k]) * 32, n, 90).view(np.int32), device=dev) for k in range(4)]
        self.d_members = torch.zeros(self.total, dtype=torch.int32, device=dev)
        self.d_off = torch.as_tensor((np.arange(self.n_agg + 1, dtype=np.int64) * CSIZE).astype(np.int32), device=dev)
        self.d_bits = torch.full((self.n_agg, CSIZE // 8), 0xFF, dtype=torch.uint8, device=dev)
        self.d_src = torch.zeros(self.n_agg, dtype=torch.int64, device=dev)
        self.d_tgt = torch.zeros(self.n_agg, dtype=torch.int64, device=dev)
        self.d_roots = torch.zeros((self.n_agg, 32), dtype=torch.uint8, device=dev)
        self.d_status = torch.zeros(self.n_agg, dtype=torch.int32, device=dev)
        self.d_kind = torch.zeros(self.total, dtype=torch.uint8, device=dev)
        self.d_conflict = torch.zeros((self.total, 2), dtype=torch.int32, device=dev)
        self.d_flagged = torch.zeros(1, dtype=torch.int32, device=dev)

    def prepare(self, cur):
        """the batch of epoch `cur` into the device arrays (not timed)"""
        torch, honest = self.torch, self.n // CSIZE
        self.d_members[:self.n] = self.pool[cur % len(self.pool)]
        if self.n_extra:
            planted = self.rng.choice(self.n, size=self.n_extra * CSIZE, replace=False).astype(np.int32)
            self.d_members[self.n:] = torch.as_tensor(planted, device=self.d_members.device)
        src = np.full(self.n_agg, cur - 1, dtype=np.int64)
        src[honest + 1::2] = cur - 3                                  # every second offending aggregate also surrounds
        roots = np.zeros((self.n_agg, 32), dtype=np.uint8)
        roots[:, 0] = cur & 0xFF
        roots[honest:, 1] = 1                                         # the offenders' other head
        self.d_src.copy_(torch.as_tensor(src))
        self.d_tgt.fill_(cur)
        self.d_roots.copy_(torch.as_tensor(roots))

    def update(self):
        self.eng.slasher_update_dev(self.d_members, self.d_off, self.d_bits, self.d_src, self.d_tgt, self.d_roots, None, self.d_status,
                                    self.d_kind, self.d_conflict, self.d_flagged)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--validators", type=int, default=1 << 20)
    ap.add_argument("--history", type=int, default=4096)
    ap.add_argument("--shares", default="0,0.001,0.05")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from pos_evolution_b200._lib import B2_ENOMEM, B2Error
    from pos_evolution_b200.engine import Engine
    assert torch.cuda.is_available(), "needs an H100: there is no CPU form of this measurement"
    n = a.validators
    assert n % CSIZE == 0
    eng = Engine(0)
    cur, history = 3 * a.history + 7, a.history
    while True:
        try:
            eng.slasher_init(n, history, PER_TARGET, cur)
            break
        except B2Error as e:
            if e.code != B2_ENOMEM or history <= 64:
                raise
            history //= 2
    result = {"validators": n, "history_epochs": history, "history_epochs_asked": a.history,
              "table_bytes": 6 * n * history + 32 * history * PER_TARGET, "aggregates_per_epoch": n // CSIZE, "committee_size": CSIZE,
              "warmup": a.warmup, "epochs": a.epochs, "rounds": a.rounds, "levels": []}
    profiled = None
    for share in [float(x) for x in a.shares.split(",")]:
        st = Stream(eng, n, share, seed=int(share * 1e6) + 1)
        planted = st.n_extra * CSIZE
        ms_rounds, adv_rounds = [], []
        for _ in range(a.rounds):
            ms, adv = [], []
            for k in range(a.warmup + a.epochs):
                cur += 1
                t_host = time.perf_counter()
                eng.slasher_advance(cur)
                adv.append((time.perf_counter() - t_host) * 1e3)
                st.prepare(cur)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                st.update()
                t1.record()
                torch.cuda.synchronize()
                assert int(st.d_flagged.item()) == planted, ("flagged", int(st.d_flagged.item()), "planted", planted)
                assert int(st.d_status.abs().sum().item()) == 0
                if k >= a.warmup:
                    ms.append(t0.elapsed_time(t1))
            ms_rounds.append(float(np.mean(ms)))
            adv_rounds.append(float(np.mean(adv[a.warmup:])))
        assert eng.guard_flags() == 0
        bits = st.total
        # per selected member: record = member index + first_id and min_span cell, each read and written; check = member index +
        # three cells + kind byte + two conflict words.  The honest span (t = s + 1) has no max_span walk.
        bytes_record, bytes_check = bits * (4 + 2 * 4) + bits // 8, bits * (4 + 3 * 2 + 1 + 8) + bits // 8
        med = float(np.median(ms_rounds))
        result["levels"].append({"offender_share": share, "planted_per_epoch": planted, "flagged_per_epoch": planted,
                                 "member_slots_per_epoch": bits, "update_ms_per_epoch": round(med, 4),
                                 "update_ms_rounds": [round(x, 4) for x in ms_rounds],
                                 "advance_ms_per_epoch_host_clock": round(float(np.median(adv_rounds)), 4),
                                 "algorithmic_bytes_record": bytes_record, "algorithmic_bytes_check": bytes_check,
                                 "algorithmic_GBps_whole_update": round((bytes_record + bytes_check) / med / 1e6, 1)})
        if profiled is None:
            profiled = st
    # the split between the kernels: device time per kernel name over five honest epochs
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                cur += 1
                eng.slasher_advance(cur)
                profiled.prepare(cur)
                profiled.update()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if "k_slasher" in ev.key:
                name = ev.key.split("k_slasher_")[1].split("(")[0]
                total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                split[name + "_ms_per_epoch"] = round(total_us / 1e3 / 5, 4)
        result["kernel_split_honest_stream"] = split or "not measured: the profiler saw no slasher kernel"
    except Exception as e:      # the profiler is an aid: without it the split is reported as missing, the event timings stand
        result["kernel_split_honest_stream"] = "not measured: %s" % e
    result["gpu"], result["power_limit"] = _card()
    eng.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
