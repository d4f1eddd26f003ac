"""Ground truth of the slasher (include/b200pos.h, b2_slasher_*): a brute force that keeps every accepted attestation of every
validator for ever and evaluates the definitions literally, quadratic in the history.  It holds no span table and no ring: only the
acceptance rule knows about the window.  The device must equal it byte for byte on status, kind and conflict targets."""
import numpy as np

OK, NOT_ACCEPTED, SOURCE_AFTER_TARGET, TARGET_AHEAD, SOURCE_EXPIRED, COLUMN_FULL, BAD_ROW = range(7)
DOUBLE, SURROUNDS, SURROUNDED = 1, 2, 4
NO_TARGET = 0xFFFFFFFF


def is_slashable(a, b) -> bool:
    """is_slashable_attestation_data (pos-evolution.md:1134-1143) on (source, target, root) triples; data_1 != data_2 <=> the roots differ"""
    return (a[2] != b[2] and a[1] == b[1]) or (a[0] < b[0] and b[1] < a[1])


class BruteSlasher:
    def __init__(self, n_validators, history_epochs, max_attestations_per_target, current_epoch=0):
        self.n, self.H, self.K, self.cur = int(n_validators), int(history_epochs), int(max_attestations_per_target), int(current_epoch)
        self.history = [[] for _ in range(self.n)]      # per validator: (source, target, root) in acceptance order, never pruned
        self.per_target = {}                             # target epoch -> aggregates accepted with it

    @property
    def low(self):
        return max(0, self.cur - self.H + 1)

    def advance(self, current_epoch):
        assert current_epoch >= self.cur
        self.cur = int(current_epoch)

    def update(self, members, off, bits, source_epoch, target_epoch, roots32, accept=None):
        """the arguments of Engine.slasher_update -> (status i32[n_agg], kind u8[total], conflict_target u32[total, 2], n_flagged)"""
        members, off = np.asarray(members, dtype=np.int64), np.asarray(off, dtype=np.int64)
        bits = np.asarray(bits, dtype=np.uint8)
        n_agg, total = len(off) - 1, int(off[-1])
        roots = [bytes(np.asarray(roots32, dtype=np.uint8).reshape(n_agg, 32)[a]) for a in range(n_agg)]
        status = np.zeros(n_agg, dtype=np.int32)
        kind = np.zeros(total, dtype=np.uint8)
        conflict = np.full((total, 2), NO_TARGET, dtype=np.uint32)

        def selected(a):
            for j in range(int(off[a + 1] - off[a])):
                if (bits[a, j >> 3] >> (j & 7)) & 1 and members[off[a] + j] < self.n:
                    yield int(off[a] + j), int(members[off[a] + j])

        for a in range(n_agg):                           # accept and record in position order
            s, t = int(source_epoch[a]), int(target_epoch[a])
            if accept is not None and not accept[a]:
                status[a] = NOT_ACCEPTED
            elif off[a + 1] < off[a] or off[a + 1] - off[a] > 8 * bits.shape[1]:
                status[a] = BAD_ROW
            elif s > t:
                status[a] = SOURCE_AFTER_TARGET
            elif t > self.cur:
                status[a] = TARGET_AHEAD
            elif s < self.low:
                status[a] = SOURCE_EXPIRED
            elif self.per_target.get(t, 0) >= self.K:
                status[a] = COLUMN_FULL
            else:
                self.per_target[t] = self.per_target.get(t, 0) + 1
                for _, v in selected(a):
                    self.history[v].append((s, t, roots[a]))
        for a in range(n_agg):                           # check against everything accepted so far, this call included
            if status[a] != OK:
                continue
            s, t = int(source_epoch[a]), int(target_epoch[a])
            for i, v in selected(a):
                hist = self.history[v]
                first = next(h for h in hist if h[1] == t)
                inner = [h[1] for h in hist if h[0] > s and h[1] < t]
                outer = [h[1] for h in hist if h[0] < s and h[1] > t]
                kind[i] = (DOUBLE if first[2] != roots[a] else 0) | (SURROUNDS if inner else 0) | (SURROUNDED if outer else 0)
                if inner:
                    conflict[i, 0] = min(inner)
                if outer:
                    conflict[i, 1] = max(outer)
        return status, kind, conflict, int(np.count_nonzero(kind))

    def slashable_validators(self):
        """validators for which is_slashable holds on SOME ordered pair of their accepted attestations"""
        return {v for v, hist in enumerate(self.history) if any(is_slashable(x, y) for x in hist for y in hist)}


def full_bits(sizes):
    """bit rows with every member selected"""
    stride = max(1, (max(sizes, default=0) + 7) // 8)
    bits = np.zeros((len(sizes), stride), dtype=np.uint8)
    for a, k in enumerate(sizes):
        bits[a, :k // 8] = 0xFF
        if k & 7:
            bits[a, k // 8] = (1 << (k & 7)) - 1
    return bits


def batch(aggregates):
    """[(members, source, target, root32 bytes)] -> the arrays of update(), every member selected"""
    members = np.array([v for m, _, _, _ in aggregates for v in m], dtype=np.uint32)
    off = np.concatenate([[0], np.cumsum([len(m) for m, _, _, _ in aggregates])]).astype(np.uint32)
    src = np.array([s for _, s, _, _ in aggregates], dtype=np.uint64)
    tgt = np.array([t for _, _, t, _ in aggregates], dtype=np.uint64)
    roots = np.frombuffer(b"".join(r for _, _, _, r in aggregates), dtype=np.uint8).reshape(len(aggregates), 32)
    return members, off, full_bits([len(m) for m, _, _, _ in aggregates]), src, tgt, roots


def root_of(tag: int) -> bytes:
    return int(tag).to_bytes(4, "little") * 8


def golden_batches(stream):
    """a stream of tests/golden/literal_slashing.json -> [(current epoch, [(members, source, target, hash_tree_root(data))])]"""
    from oracle import spec as S
    out = []
    for call in stream["calls"]:
        aggs = []
        for a in call["aggregates"]:
            data = S.AttestationData(slot=a["slot"], index=a["index"], beacon_block_root=bytes.fromhex(a["beacon_block_root"]),
                                     source=S.Checkpoint(a["source"], bytes.fromhex(a["source_root"])),
                                     target=S.Checkpoint(a["target"], bytes.fromhex(a["target_root"])))
            aggs.append((a["members"], a["source"], a["target"], S.hash_tree_root_attestation_data(data)))
        out.append((call["current_epoch"], aggs))
    return out
