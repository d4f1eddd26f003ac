"""What Electra block attestations cost: 2^20 validators on the mainnet preset (64 committees of 512 a slot), the committees of two epochs
from two random permutations, attestations signed through Engine.sign with the arithmetic-progression keys.  Each aggregate names about 95 %
of its slot's 64 committees (committee_bits) with about 95 % of their bits, so it covers about 29 000 validators in a row of 32 768.

    python tools/block_attestations_electra_bench.py [--rounds 7]
    python tools/block_attestations_electra_bench.py --profile     # one torch.profiler pass per load: the split over the kernels

Two loads: one block of 8 aggregates, and 32 blocks x 8 (a full epoch).  Reported per load:
  device_ms       device time of one Engine.block_attestations_electra_dev call (CUDA events around the call, median and range)
  fav_warp_ms     device time of the same FastAggregateVerify (the same padded member and bit rows, messages and signatures) through
                  b2_fast_aggregate_verify_dev, whose key sum gives one warp to each aggregate (median and range)
With --profile, the kernel split of one call and of one warp-per-aggregate FastAggregateVerify: the split key sum (k_g1_gather_tma over
the chunks, then k_bae_pk_combine) against k_g1_gather_tma with one warp per aggregate.
Every aggregate verifies on both paths.  Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (sets CUDA_DEVICE_MAX_CONNECTIONS before the first CUDA call)
import numpy as np  # noqa: E402
import block_attestations_electra_oracle as E  # noqa: E402
from epoch_discount_bench import _card  # noqa: E402
from sync_messages_bench import _h  # noqa: E402

SPE, CPS, SIZE, M, MAX_VPC, EP = 32, 64, 512, 64, 2048, 3
START, PART = EP * SPE, 0.95
DOMAINS = _h(b"attester e-1") + _h(b"attester e")
JUSTIFIED = (EP - 2).to_bytes(8, "little") + _h(b"j-prev") + (EP - 1).to_bytes(8, "little") + _h(b"j-cur")
ROOTS = [_h(b"root" + s.to_bytes(8, "little")) for s in range(2 * SPE)]


class Load:
    """n_blocks blocks at START .. with 8 aggregates each of the 8 slots before the block, signed; the call's device arguments and the
    padded rows the warp-per-aggregate FastAggregateVerify takes"""

    def __init__(self, eng, sk0, delta, members, off, n_blocks, rng):
        import torch
        dev = torch.device("cuda", 0)
        wires, sks, msgs, rows, brows = [], [], [], [], []
        R = SIZE * CPS                                  # row_max: every row padded to it
        for k in range(n_blocks):
            s = START + k
            for j in range(8):
                slot = s - 1 - j
                ep = slot // SPE
                picks = [i for i in range(CPS) if rng.random() < PART]
                c0 = (0 if ep == EP - 1 else SPE * CPS) + (slot - ep * SPE) * CPS
                bits, sel, row = [], [], []
                for i in picks:
                    com = members[off[c0 + i]:off[c0 + i + 1]]
                    b = rng.random(len(com)) < PART
                    bits.append(b)
                    sel.append(com[b])
                    row.append(com)
                bits, sel, row = np.concatenate(bits), np.concatenate(sel), np.concatenate(row)
                src = JUSTIFIED[40:80] if ep == EP else JUSTIFIED[0:40]
                d = E.data128(slot, 0, ROOTS[slot + SPE - START], int.from_bytes(src[:8], "little"), src[8:], ep, ROOTS[SPE if ep == EP else 0])
                msgs.append(E.signing_root(d, DOMAINS[32:] if ep == EP else DOMAINS[:32]))
                sks.append((int(sel.astype(object).sum()) * delta + len(sel) * sk0) % bench.R_ORDER)
                wires.append((bits, d, E.committee_bits_of(picks, M)))
                rows.append(np.concatenate([row, np.zeros(R - len(row), np.uint32)]))
                brows.append(np.packbits(np.concatenate([bits, np.zeros(R - len(bits), bool)]).astype(np.uint8), bitorder="little"))
        sigs = eng.sign(sks, np.arange(len(sks), dtype=np.uint32),
                        np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32))
        enc = [E.encode(b.tolist(), d, bytes(sig), cb) for (b, d, cb), sig in zip(wires, sigs)]
        n = len(enc)
        woff = np.concatenate([[0], np.cumsum([len(w) for w in enc])]).astype(np.uint32)
        T = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dtype=dt).copy()).to(dev)      # noqa: E731
        self.n, self.n_blocks = n, n_blocks
        self.args = [T(np.frombuffer(b"".join(enc), np.uint8), np.uint8), T(woff, np.uint32), T(np.arange(0, n + 1, 8), np.uint32),
                     T(START + np.arange(n_blocks), np.uint64), T(members, np.uint32), T(off, np.uint32), CPS, CPS,
                     T(np.frombuffer(b"".join(ROOTS), np.uint8), np.uint8), JUSTIFIED, DOMAINS, SPE, 1, M, MAX_VPC, SIZE * CPS, 10**9, 977]
        self.fav = [T(np.stack(rows).reshape(-1), np.uint32), T(np.arange(0, n + 1) * R, np.uint32), T(np.stack(brows), np.uint8),
                    T(np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32), np.uint8), T(np.stack([np.frombuffer(bytes(x), np.uint8) for x in sigs]), np.uint8),
                    torch.zeros(n, dtype=torch.uint8, device=dev)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    n = bench.N_VAL
    sk0 = int.from_bytes(_h(b"b200pos/sk0"), "big") % (bench.R_ORDER >> 1) or 1
    delta = int.from_bytes(_h(b"b200pos/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), dtype=np.uint32).reshape(n, 8)
    eng.registry_load(eng.sk_to_pk(sk8), np.full(n, 32 * 10**9, np.uint64))
    rng = np.random.default_rng(3)
    members = np.concatenate([rng.permutation(n), rng.permutation(n)]).astype(np.uint32)      # epochs e - 1 and e
    off = (np.arange(2 * SPE * CPS + 1) * SIZE).astype(np.uint32)
    zeros = np.zeros(n, np.uint8)
    out = {"tool": "block_attestations_electra_bench", "validators": n, "committees_per_slot": CPS, "committee_size": SIZE}
    for n_blocks in (1, 32):
        L = Load(eng, sk0, delta, members, off, n_blocks, rng)

        def call():
            eng.participation_load(0, zeros)
            eng.participation_load(1, zeros)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = eng.block_attestations_electra_dev(*L.args)
            e1.record()
            torch.cuda.synchronize()
            return r, e0.elapsed_time(e1)

        def fav():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.fast_aggregate_verify_dev(*L.fav)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        r, _ = call()                                                             # warm-up
        fav()
        assert not r.status.cpu().numpy().any() and int(r.n_applied.cpu()[0]) == n_blocks, "every aggregate is valid"
        assert L.fav[-1].cpu().numpy().all(), "every aggregate verifies on the warp-per-aggregate path"
        key = "%d_blocks" % n_blocks
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            split = {}
            for name, fn in (("call", lambda: call()), ("fav_warp", fav)):
                eng.participation_load(0, zeros)
                eng.participation_load(1, zeros)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn()
                part = {}
                for ev in prof.key_averages():
                    if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                        part[ev.key] = round(ev.device_time_total / 1000.0, 3)
                split[name] = dict(sorted(part.items(), key=lambda kv: -kv[1]))
            out["profile_ms_" + key] = split
            continue
        times, ftimes = [], []
        for _ in range(args.rounds):
            times.append(call()[1])
            ftimes.append(fav())
        out[key] = {"aggregates": L.n, "device_ms": round(float(np.median(times)), 3), "device_ms_range": [round(min(times), 3), round(max(times), 3)],
                    "fav_warp_ms": round(float(np.median(ftimes)), 3), "fav_warp_ms_range": [round(min(ftimes), 3), round(max(ftimes), 3)]}
    out["gpu"], out["power_limit"] = _card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
