"""Block-packing oracles (b2_pack_attestations, include/b200pos.h): the literal global greedy of the contract, and an independent
per-committee greedy + merge (numpy, fast enough for mainnet-size pools).  Python ints throughout the literal form.

A pool is a dict:
  members, off, table     committees k: members[off[k]:off[k+1]], participation table 0 (current) / 1 (previous)
  comm, data, mask        per candidate (pool order): committee, data id, flag mask
  bits                    uint8[n_cand, stride] bit rows (bits at or past the committee size are ignored)
  ok                      per candidate: the signature decodes
  eff                     effective balance per validator
  part                    (current, previous) participation bytes per validator
  inc, per_inc, max_out
A packing is a list of picks (committee, data id, union row as int, gain, constituents tuple) in pick order."""
import numpy as np

WEIGHTS = (14, 26, 14)


def _row(pool, c):
    k = pool["comm"][c]
    size = int(pool["off"][k + 1]) - int(pool["off"][k])
    return int.from_bytes(bytes(np.asarray(pool["bits"][c], dtype=np.uint8)), "little") & ((1 << size) - 1)


def fold(pool):
    """step 2: first fit per data id in pool order -> list of [committee, data, mask, union row, constituents] in creation order"""
    folded, by_data = [], {}
    for c in range(len(pool["comm"])):
        if not pool["ok"][c]:
            continue
        d, r = int(pool["data"][c]), _row(pool, c)
        for f in by_data.get(d, []):
            if folded[f][3] & r == 0:
                folded[f][3] |= r
                folded[f][4].append(c)
                break
        else:
            by_data.setdefault(d, []).append(len(folded))
            folded.append([int(pool["comm"][c]), d, int(pool["mask"][c]) & 7, r, [c]])
    return folded


def _unit(pool, v):
    return (int(pool["eff"][v]) // pool["inc"]) * pool["per_inc"]


def gain(pool, f, part):
    k, _, mask, row, _ = f
    t, base, g = int(pool["table"][k]), int(pool["off"][k]), 0
    j = 0
    while row >> j:
        if (row >> j) & 1:
            v = int(pool["members"][base + j])
            for fl in range(3):
                if (mask >> fl) & 1 and not (part[t][v] >> fl) & 1:
                    g += _unit(pool, v) * WEIGHTS[fl]
        j += 1
    return g


def pack_literal(pool):
    """The contract as written: every step recomputes every gain and takes the largest (lowest committee, then lowest folded number)."""
    folded = fold(pool)
    part = [list(int(x) for x in pool["part"][0]), list(int(x) for x in pool["part"][1])]
    out = []
    for _ in range(pool["max_out"]):
        best, bi = 0, None
        for i, f in enumerate(folded):
            g = gain(pool, f, part)
            if g > best or (g == best and g > 0 and (f[0], f[4][0]) < (folded[bi][0], folded[bi][4][0])):
                best, bi = g, i
        if bi is None:
            break
        k, d, mask, row, src = folded[bi]
        t, base = int(pool["table"][k]), int(pool["off"][k])
        for j in range(row.bit_length()):
            if (row >> j) & 1:
                part[t][int(pool["members"][base + j])] |= mask
        out.append((k, d, row, best, tuple(src)))
    return out


def pack_per_committee(pool):
    """Each committee's own greedy (at most min(max_out, folded) steps, stop at gain 0), merged by (gain desc, committee, step)."""
    folded = fold(pool)
    by_comm = {}
    for f in folded:
        by_comm.setdefault(f[0], []).append(f)
    wtab = np.array([sum(w for b, w in enumerate(WEIGHTS) if (m >> b) & 1) for m in range(8)], dtype=np.uint64)
    entries = []
    for k, fs in by_comm.items():
        lo, hi = int(pool["off"][k]), int(pool["off"][k + 1])
        mem = np.asarray(pool["members"][lo:hi], dtype=np.int64)
        unit = (np.asarray(pool["eff"], dtype=np.uint64)[mem] // np.uint64(pool["inc"])) * np.uint64(pool["per_inc"])
        part = np.asarray(pool["part"][int(pool["table"][k])], dtype=np.uint8)[mem].copy()
        nb = (hi - lo + 7) // 8
        rows = np.stack([np.unpackbits(np.frombuffer(f[3].to_bytes(nb, "little"), dtype=np.uint8), bitorder="little")[:hi - lo] for f in fs]).astype(bool)
        masks = np.array([f[2] for f in fs], dtype=np.uint8)
        for step in range(min(pool["max_out"], len(fs))):
            w = wtab[masks[:, None] & ~part[None, :]]
            gains = [int(x) for x in (np.where(rows, w * unit[None, :], np.uint64(0))).sum(axis=1, dtype=np.uint64)]
            i = max(range(len(fs)), key=lambda i: (gains[i], -i))
            if gains[i] == 0:
                break
            part[rows[i]] |= masks[i]
            entries.append((-gains[i], k, step, fs[i]))
    entries.sort(key=lambda e: e[:3])
    return [(f[0], f[1], f[3], -g, tuple(f[4])) for g, _, _, f in entries[:pool["max_out"]]]


def row_bytes(row: int, stride: int) -> bytes:
    return row.to_bytes(stride, "little")


def random_pool(seed, n_val=256, comms=(4, 4), n_cand=60, max_out=8, tie_heavy=False, stride=None, bad_frac=0.0, singles=0.2):
    """A seeded pool: comms[t] disjoint committees of table t (the two tables shuffled independently, so they overlap), a few votes
    (data ids) per committee, aggregates, single-bit attestations and -- with tie_heavy -- equal balances, no prior participation and
    rows copied between committees of equal size and within a committee."""
    rng = np.random.default_rng(seed)
    eff = np.full(n_val, 32 * 10**9, dtype=np.uint64) if tie_heavy else rng.choice([16, 24, 31, 32, 32], size=n_val).astype(np.uint64) * np.uint64(10**9)
    part = [np.zeros(n_val, dtype=np.uint8) if tie_heavy else (rng.integers(0, 8, size=n_val) * (rng.random(n_val) < 0.3)).astype(np.uint8)
            for _ in range(2)]
    members, off, table = [], [0], []
    for t, nk in enumerate(comms):
        perm = rng.permutation(n_val)
        size = n_val // max(nk, 1)
        for k in range(nk):
            members += [int(x) for x in perm[k * size:(k + 1) * size]]
            off.append(len(members))
            table.append(t)
    K = len(table)
    sizes = [off[k + 1] - off[k] for k in range(K)]
    stride = stride or max(1, (max(sizes, default=1) + 7) // 8)
    votes = {}
    comm, data, mask, rows, ok = [], [], [], [], []
    for c in range(n_cand):
        k = int(rng.integers(0, K))
        v = (k, int(rng.integers(0, 2 if tie_heavy else 3)))
        if v not in votes:
            votes[v] = (len(votes), 7 if tie_heavy else int(rng.integers(1, 8)))
        d, m = votes[v]
        r = rng.random()
        if r < singles:
            row = np.zeros(sizes[k], dtype=np.uint8)
            row[int(rng.integers(0, sizes[k]))] = 1
        elif tie_heavy and rows and r < 0.6:
            src = int(rng.integers(0, len(rows)))
            row = np.unpackbits(rows[src], bitorder="little")[:sizes[k]] if sizes[comm[src]] == sizes[k] else (rng.random(sizes[k]) < 0.5)
        else:
            row = rng.random(sizes[k]) < rng.choice([0.2, 0.5, 0.9])
        b = np.zeros(stride, dtype=np.uint8)
        packed = np.packbits(np.asarray(row, dtype=np.uint8), bitorder="little")
        b[:len(packed)] = packed
        if r > 0.9 and 8 * stride > sizes[k]:                       # junk past the committee size: ignored
            b[-1] |= 0x80
        comm.append(k)
        data.append(d)
        mask.append(m)
        rows.append(b)
        ok.append(bool(rng.random() >= bad_frac))
    return {"members": np.asarray(members, dtype=np.uint32), "off": np.asarray(off, dtype=np.uint32), "table": np.asarray(table, dtype=np.uint8),
            "comm": np.asarray(comm, dtype=np.uint32), "data": np.asarray(data, dtype=np.uint32), "mask": np.asarray(mask, dtype=np.uint8),
            "bits": np.asarray(rows, dtype=np.uint8).reshape(n_cand, stride), "ok": ok, "eff": eff, "part": part,
            "inc": 10**9, "per_inc": 1234 if not tie_heavy else 1000, "max_out": max_out}
