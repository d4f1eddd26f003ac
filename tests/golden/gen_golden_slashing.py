#!/usr/bin/env python3
"""Generates tests/golden/literal_slashing.json by EXECUTING THE REFERENCE'S OWN is_slashable_attestation_data
(pos-evolution.md:1134-1143, loaded by tests/ref_blocks.py -- never copied) over all ordered pairs of seeded attestation streams.
A stream is a sequence of calls (current epoch + aggregates: members and the five AttestationData fields); the file stores the streams
and, per stream, the ordered pairs (i, j) of aggregates, numbered in stream order, whose data the reference calls slashable.
tests/test_oracle_slashing.py replays it against tests/slasher_oracle.py and Spec.is_slashable_attestation_data, tests/test_gpu_slasher.py
against the device.  It writes no other file.
Run where a copy of the reference is available:  POS_EVOLUTION_MD=<path>/pos-evolution.md python tests/golden/gen_golden_slashing.py"""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ref_blocks  # noqa: E402
from oracle import spec as S  # noqa: E402

N_VALIDATORS = 16
HISTORY_EPOCHS = 16


def stream(seed, n_calls, offender_rate):
    """calls with a rising current epoch; honest aggregates vote (cur - 1, cur), offenders anything inside the window, sometimes the
    same epochs with another head (double vote) and sometimes the very same data again (not slashable)"""
    rng = random.Random(seed)
    calls, cur, seen = [], rng.randrange(0, 3), []
    for _ in range(n_calls):
        cur += rng.choice([0, 1, 1, 2])
        low = max(0, cur - HISTORY_EPOCHS + 1)
        aggs = []
        for _ in range(rng.randrange(1, 5)):
            members = sorted(rng.sample(range(N_VALIDATORS), rng.randrange(1, 6)))
            if seen and rng.random() < 0.15:
                d = dict(rng.choice(seen))                               # identical data re-submitted
            else:
                if rng.random() < offender_rate:
                    s = rng.randrange(low, cur + 1)
                    t = rng.randrange(s, cur + 1)
                else:
                    s, t = max(low, cur - 1), cur
                d = dict(slot=8 * t + rng.randrange(8), index=rng.randrange(2), beacon_block_root=bytes([rng.randrange(3)]) * 32,
                         source=s, source_root=bytes([0x50 + s % 7]) * 32, target=t, target_root=bytes([0xA0 + t % 7]) * 32)
            seen.append(d)
            aggs.append(dict(d, members=members))
        calls.append({"current_epoch": cur, "aggregates": aggs})
    return calls


def data_of(d):
    return S.AttestationData(slot=d["slot"], index=d["index"], beacon_block_root=d["beacon_block_root"],
                             source=S.Checkpoint(d["source"], d["source_root"]), target=S.Checkpoint(d["target"], d["target_root"]))


def main():
    assert ref_blocks.available(), "set POS_EVOLUTION_MD to the reference's pos-evolution.md"
    ns = ref_blocks.exec_functions(["is_slashable_attestation_data"], dict(AttestationData=S.AttestationData))
    predicate = ns["is_slashable_attestation_data"]
    out = {"generator": "tests/golden/gen_golden_slashing.py (reference block executed literally)", "n_validators": N_VALIDATORS,
           "history_epochs": HISTORY_EPOCHS, "streams": []}
    for seed, n_calls, rate in ((1, 12, 0.0), (2, 20, 0.3), (3, 30, 0.6), (4, 40, 0.15)):
        calls = stream(seed, n_calls, rate)
        flat = [data_of(a) for c in calls for a in c["aggregates"]]
        pairs = [[i, j] for i, x in enumerate(flat) for j, y in enumerate(flat) if predicate(x, y)]
        for c in calls:
            for a in c["aggregates"]:
                for k in ("beacon_block_root", "source_root", "target_root"):
                    a[k] = a[k].hex()
        out["streams"].append({"seed": seed, "calls": calls, "slashable_pairs": pairs})
    with open(os.path.join(HERE, "literal_slashing.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote literal_slashing.json:", [len(s["slashable_pairs"]) for s in out["streams"]], "slashable pairs")


if __name__ == "__main__":
    main()
