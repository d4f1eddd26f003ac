#!/usr/bin/env python3
"""Generates tests/golden/literal_sync.json by EXECUTING THE REFERENCE'S OWN compute_sync_committee_period and
is_assigned_to_sync_committee (pos-evolution.md:564-587, loaded by tests/ref_blocks.py -- never copied) on minimal states that carry a
sync committee: a committee with a duplicate member, queries in the current and the next period, and the assertion for an epoch two
periods ahead.  tests/test_oracle_sync.py replays the file against tests/sync_oracle.py.  It writes no other file, so the fixtures of
tests/golden/gen_golden.py stay as they are.
Run where a copy of the reference is available:  POS_EVOLUTION_MD=<path>/pos-evolution.md python tests/golden/gen_golden_sync.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import literal  # noqa: E402
import ref_blocks  # noqa: E402
import scenarios  # noqa: E402
import sync_oracle as SO  # noqa: E402

N_VALIDATORS = 64


def committees(pks, size):
    """(current, next) pubkey lists: current repeats validator 3 and skips validator 4; next is a different, shifted selection"""
    cur = [pks[(5 * i) % N_VALIDATORS] for i in range(size)]
    cur[1] = pks[3]
    cur[2] = pks[3]
    nxt = [pks[(7 * i + 11) % N_VALIDATORS] for i in range(size)]
    return cur, nxt


def cases(spec):
    """[(state slot, epoch queried)]: each period boundary from both sides, the next period, and two periods ahead"""
    per = spec.EPOCHS_PER_SYNC_COMMITTEE_PERIOD
    spe = spec.p.SLOTS_PER_EPOCH
    out = []
    for state_epoch in (0, per - 1, per, 2 * per + 3):
        for d in (0, 1, per - 1 - state_epoch % per, per - state_epoch % per, 2 * per - state_epoch % per - 1, 2 * per):
            out.append((state_epoch * spe + 1, state_epoch + d))
    return out


def main():
    assert ref_blocks.available(), "set POS_EVOLUTION_MD to the reference's pos-evolution.md"
    pks = scenarios.pubkeys(N_VALIDATORS)
    spec, state = scenarios.minimal_state(N_VALIDATORS, slot=9, pks=pks)
    spec = SO.SyncSpec(spec.p)
    ns = literal.namespace(spec)
    ns.update(EPOCHS_PER_SYNC_COMMITTEE_PERIOD=spec.EPOCHS_PER_SYNC_COMMITTEE_PERIOD, ValidatorIndex=int, BeaconState=object)
    ref_blocks.exec_functions(["compute_sync_committee_period", "is_assigned_to_sync_committee"], ns)
    cur, nxt = committees(pks, spec.SYNC_COMMITTEE_SIZE)
    state.current_sync_committee = SO.SyncCommittee(cur, b"")
    state.next_sync_committee = SO.SyncCommittee(nxt, b"")
    out = {"preset": "minimal", "n_validators": N_VALIDATORS, "generator": "tests/golden/gen_golden_sync.py (reference blocks executed literally)",
           "current_sync_committee": [pks.index(p) for p in cur], "next_sync_committee": [pks.index(p) for p in nxt],
           "period": {str(e): int(ns["compute_sync_committee_period"](e)) for e in range(0, 40)}, "assigned": []}
    for slot, epoch in cases(spec):
        state.slot = slot
        try:
            res = [bool(ns["is_assigned_to_sync_committee"](state, epoch, v)) for v in range(N_VALIDATORS)]
        except AssertionError:
            res = "assert"
        out["assigned"].append({"state_slot": slot, "epoch": epoch, "result": res})
    with open(os.path.join(HERE, "literal_sync.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote literal_sync.json")


if __name__ == "__main__":
    main()
