"""What process_attestation costs for one epoch of blocks: 2^20 validators (mainnet preset: 64 committees of 512 per slot), 32 blocks of
128 aggregates each (block k at slot start(e) + k carries the 64 aggregates of each of the two slots before it, about 95 % of each
committee set), every signature valid (Engine.sign with each aggregate's summed secret key of the arithmetic-progression keys).

    python tools/block_attestations_bench.py [--rounds 5] [--spec-blocks 1]
    python tools/block_attestations_bench.py --profile     # one torch.profiler pass: the split over the call's kernels

Reported:
  device_ms        device time of one Engine.block_attestations_dev call over the 32 blocks (CUDA events, median and range over the
                   rounds; the participation tables are reloaded, untimed, before each round);
  spec_block_s     wall time of Spec.process_attestations on the same state and the same attestations, block by block, for the first
                   --spec-blocks blocks (that path checks, builds each IndexedAttestation and loads / reads the participation tables in
                   Python per block); per block, so the two figures are compared per block and not extrapolated.
Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(ROOT)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402
from epoch_discount_bench import _card  # noqa: E402

EPOCH = 3
PARTICIPATION = 0.95


def _h(b):
    return hashlib.sha256(b).digest()


def world(eng, PS):
    """the state (2^20 validators, chain roots for epochs e - 1 and e) and the 32 blocks of epoch e"""
    n = bench.N_VAL
    p = PS.MAINNET
    spe = p.SLOTS_PER_EPOCH
    sk0 = int.from_bytes(_h(b"b200pos/sk0"), "big") % (bench.R_ORDER >> 1) or 1
    delta = int.from_bytes(_h(b"b200pos/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), dtype=np.uint32).reshape(n, 8)
    pk = eng.sk_to_pk(sk8)
    validators = [PS.Validator(pk[i].tobytes(), 32 * 10**9) for i in range(n)]
    start = EPOCH * spe
    block_roots = [_h(b"root" + s.to_bytes(8, "little")) for s in range(p.SLOTS_PER_HISTORICAL_ROOT)]
    state = PS.BeaconState(slot=start, fork=PS.Fork(), genesis_validators_root=bytes(32), validators=validators, balances=[32 * 10**9] * n,
                           randao_mixes=[_h(b"mix" + i.to_bytes(8, "little")) for i in range(p.EPOCHS_PER_HISTORICAL_VECTOR)],
                           block_roots=block_roots, previous_epoch_participation=[0] * n, current_epoch_participation=[0] * n,
                           previous_justified_checkpoint=PS.Checkpoint(EPOCH - 2, _h(b"j-prev")),
                           current_justified_checkpoint=PS.Checkpoint(EPOCH - 1, _h(b"j-cur")))
    return state, sk0, delta


def blocks_of(eng, pspec, PS, state, sk0, delta, rng):
    p = pspec.p
    spe = p.SLOTS_PER_EPOCH
    start = EPOCH * spe
    cur = EPOCH
    blocks, sks, msgs = [], [], []
    committees = {E: pspec.epoch_committees(state, E) for E in (EPOCH - 1, EPOCH)}
    for k in range(spe):
        s = start + k
        atts = []
        for ds in (1, 2):
            slot = s - ds
            E = slot // spe
            members, off, cps = committees[E]
            for i in range(cps):
                c = (slot - E * spe) * cps + i
                com = members[off[c]:off[c + 1]]
                bits = rng.random(len(com)) < PARTICIPATION
                src = state.current_justified_checkpoint if E == cur else state.previous_justified_checkpoint
                data = PS.AttestationData(slot, i, bytes(state.block_roots[slot % p.SLOTS_PER_HISTORICAL_ROOT]), src,
                                          PS.Checkpoint(E, bytes(state.block_roots[(E * spe) % p.SLOTS_PER_HISTORICAL_ROOT])))
                sel = com[bits].astype(object)
                sks.append((int(sel.sum()) * delta + len(sel) * sk0) % bench.R_ORDER)
                msgs.append(pspec.compute_signing_root(data, pspec.get_domain(state, PS.DOMAIN_BEACON_ATTESTER, E)))
                atts.append(PS.Attestation(bits.tolist(), data, None))
        blocks.append(PS.BlockAttestations(s, 0, bytes(state.block_roots[s % p.SLOTS_PER_HISTORICAL_ROOT]), atts))      # the chain's own roots
    sk8 = np.frombuffer(b"".join(v.to_bytes(32, "little") for v in sks), dtype=np.uint32).reshape(-1, 8)
    sigs = eng.sign(sk8, np.arange(len(sks), dtype=np.uint32), np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32))
    j = 0
    for b in blocks:
        for a in b.attestations:
            a.signature = sigs[j].tobytes()
            j += 1
    return blocks


def device_inputs(pspec, state, blocks):
    """Spec.block_attestations_inputs (what Spec.process_block_attestations passes), its arrays on the device, and the outputs"""
    import torch
    a = pspec.block_attestations_inputs(state, blocks)
    T = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()      # noqa: E731
    for k, dt in (("woff", np.uint32), ("block_off", np.uint32), ("block_slot", np.uint64), ("members", np.uint32), ("off", np.uint32),
                  ("chain_roots", np.uint8)):
        a[k] = T(a[k], dt)
    a["wire"] = T(np.frombuffer(a["wire"], np.uint8), np.uint8)
    n, nb = a["woff"].numel() - 1, a["block_off"].numel() - 1
    outs = [torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda"),
            torch.zeros(n, dtype=torch.uint64, device="cuda"), torch.zeros(nb, dtype=torch.int32, device="cuda"),
            torch.zeros(nb, dtype=torch.uint32, device="cuda"), torch.zeros(nb, dtype=torch.uint64, device="cuda"),
            torch.zeros(1, dtype=torch.uint32, device="cuda")]
    return a, outs


def call(eng, a, outs):
    eng.block_attestations_dev(a["wire"], a["woff"], a["block_off"], a["block_slot"], a["members"], a["off"], a["cps_prev"], a["cps_cur"],
                               a["chain_roots"], a["justified80"], a["domains64"], a["slots_per_epoch"], a["min_inclusion_delay"],
                               a["bits_stride"], a["increment"], a["base_reward_per_increment"], *outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--spec-blocks", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    pspec = PS.Spec(PS.MAINNET, engine=eng)
    state, sk0, delta = world(eng, PS)
    blocks = blocks_of(eng, pspec, PS, state, sk0, delta, np.random.default_rng(5))
    d, outs = device_inputs(pspec, state, blocks)
    pspec.sync_registry(state)
    zeros = np.zeros(bench.N_VAL, np.uint8)

    def fresh():
        eng.participation_load(0, zeros)
        eng.participation_load(1, zeros)

    fresh()
    call(eng, d, outs)                  # warm-up: module load, scratch allocation
    torch.cuda.synchronize()
    status, block_status = outs[0].cpu().numpy(), outs[3].cpu().numpy()
    assert int(outs[6].cpu()[0]) == len(blocks) and not status.any() and not block_status.any(), "every block must apply"
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        fresh()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(eng, d, outs)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                split[ev.key] = round(ev.device_time_total / 1000.0, 3)
        name, power = _card()
        print(json.dumps({"tool": "block_attestations_bench", "profile_ms": dict(sorted(split.items(), key=lambda kv: -kv[1])), "gpu": name,
                          "power_limit": power}))
        return
    times = []
    for _ in range(args.rounds):
        fresh()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(eng, d, outs)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    spec_s = []
    for b in blocks[:args.spec_blocks]:
        state.slot = b.slot
        t0 = time.perf_counter()
        pspec.process_attestations(state, b.attestations)
        spec_s.append(time.perf_counter() - t0)
    name, power = _card()
    print(json.dumps({"tool": "block_attestations_bench", "validators": bench.N_VAL, "blocks": len(blocks),
                      "aggregates": int(sum(len(b.attestations) for b in blocks)), "device_ms": round(float(np.median(times)), 3),
                      "device_ms_range": [round(min(times), 3), round(max(times), 3)],
                      "device_ms_per_block": round(float(np.median(times)) / len(blocks), 3),
                      "spec_block_s": [round(x, 3) for x in spec_s], "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
