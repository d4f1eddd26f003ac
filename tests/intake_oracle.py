"""Host oracle of the attestation intake (include/b200pos.h, b2_attestation_intake): one epoch of unaggregated Attestations on the wire,
checked as process_attestation (pos-evolution.md:724-730) and validate_on_attestation (upstream fork-choice spec v1.2.0, :963-979) require
against a block store, one kept per committee position, grouped by AttestationData into the vote form's inputs.

intake_plain restates the contract attestation by attestation over oracle.spec containers, a block dict and oracle.spec's get_ancestor
and hash_tree_root_attestation_data; intake_numpy computes the same for fixed-length records with array operations, for epochs of 2^20."""
import hashlib
import types

import numpy as np

from oracle.spec import AttestationData, BeaconBlock, Checkpoint, Spec, hash_tree_root_attestation_data
from oracle.ssz import compute_signing_root_from_object_root

FIXED = 228
NONE = 0xFFFFFFFF
Result = types.SimpleNamespace


def data_from_bytes(d: bytes) -> AttestationData:
    u = lambda o: int.from_bytes(d[o:o + 8], "little")      # noqa: E731
    return AttestationData(u(0), u(8), bytes(d[16:48]), Checkpoint(u(48), bytes(d[56:88])), Checkpoint(u(88), bytes(d[96:128])))


def block_store(parent, slot, roots):
    """the tree (parent ids, slots, 32-byte roots; block 0 the root) as store.blocks and the root -> id map; the root's parent_root names
    no block, so a walk past it fails as get_ancestor does on a pruned store"""
    roots = [bytes(r) for r in np.asarray(roots, dtype=np.uint8).reshape(-1, 32)]
    outside = b"\xff" * 32
    assert outside not in roots
    blocks = {r: BeaconBlock(int(slot[b]), outside if b == 0 else roots[int(parent[b])]) for b, r in enumerate(roots)}
    ids = {}
    for b, r in enumerate(roots):
        ids.setdefault(r, b)
    return blocks, ids


def _decode(w: bytes, max_bits: int):
    """(status 1-3 or 0, bits)"""
    if len(w) < FIXED or int.from_bytes(w[:4], "little") != FIXED:
        return 1, None
    b = w[FIXED:]
    if len(b) == 0 or b[-1] == 0:
        return 2, None
    n = 8 * (len(b) - 1) + b[-1].bit_length() - 1
    if n > max_bits:
        return 3, None
    return 0, [bool((b[i >> 3] >> (i & 7)) & 1) for i in range(n)]


def intake_plain(wires, off, epoch, current_slot, domain, committees_per_slot, slots_per_epoch, bits_stride, blocks, ids):
    """wires: one encoding per attestation (list order); off: the committee layout; blocks / ids: block_store's.  Every vote row, not
    only the first max_votes."""
    store = types.SimpleNamespace(blocks=blocks)
    start = epoch * slots_per_epoch
    status, kept = [], {}
    for i, w in enumerate(wires):
        w = bytes(w)
        st, bits = _decode(w, 8 * bits_stride)
        if st == 0 and sum(bits) != 1:
            st = 4
        if st == 0:
            data = data_from_bytes(w[4:132])
            if not start <= data.slot < start + slots_per_epoch or data.index >= committees_per_slot:
                st = 6
            else:
                c = (data.slot - start) * committees_per_slot + data.index
                p = bits.index(True)
                if len(bits) != int(off[c + 1]) - int(off[c]):
                    st = 5
                elif data.target.epoch != epoch:
                    st = 7
                elif current_slot < data.slot + 1:
                    st = 8
                elif data.beacon_block_root not in blocks:
                    st = 9
                elif data.target.root not in blocks:
                    st = 10
                elif blocks[data.beacon_block_root].slot > data.slot:
                    st = 11
                else:
                    try:
                        anc = Spec.get_ancestor(None, store, data.beacon_block_root, start)
                    except KeyError:
                        anc = None
                    if anc != data.target.root:
                        st = 12
                    elif (c, p) in kept:
                        st = 13
                    else:
                        kept[(c, p)] = (w[4:132], w[132:228], data)
        status.append(st)
    n_c = len(off) - 1
    n_sig = int(off[-1])
    vote = np.full(n_sig, NONE, dtype=np.uint32)
    sigs = np.zeros((n_sig, 96), dtype=np.uint8)
    vote_off, rows = [0], []
    for c in range(n_c):
        groups = {}
        for p in range(int(off[c + 1]) - int(off[c])):
            if (c, p) in kept:
                groups.setdefault(kept[(c, p)][0], []).append(p)      # positions ascend: a group's first is its smallest
        order = sorted(groups, key=lambda d: groups[d][0])
        for d in order:
            v = len(rows)
            data = kept[(c, groups[d][0])][2]
            msg = compute_signing_root_from_object_root(hash_tree_root_attestation_data(data), domain)
            rows.append((d, msg, data.source.epoch, data.target.epoch, ids[data.beacon_block_root]))
            for p in groups[d]:
                vote[int(off[c]) + p] = v
                sigs[int(off[c]) + p] = np.frombuffer(kept[(c, p)][1], dtype=np.uint8)
        if not order:
            rows.append((bytes(128), bytes(32), 0, 0, 0))
        vote_off.append(len(rows))
    return _result(np.array(status, dtype=np.int32), vote, np.array(vote_off, dtype=np.int64), sigs, rows)


def _result(status, vote, vote_off, sigs, rows):
    n = len(rows)
    return Result(status=status, vote=vote, vote_off=vote_off, sigs=sigs,
                  data128=np.frombuffer(b"".join(r[0] for r in rows), dtype=np.uint8).reshape(n, 128),
                  msgs=np.frombuffer(b"".join(r[1] for r in rows), dtype=np.uint8).reshape(n, 32),
                  source_epoch=np.array([r[2] for r in rows], dtype=np.uint64), target_epoch=np.array([r[3] for r in rows], dtype=np.uint64),
                  block_idx=np.array([r[4] for r in rows], dtype=np.uint32))


_POP = np.array([bin(x).count("1") for x in range(256)], dtype=np.uint8)
_TOP = np.array([max(x.bit_length() - 1, 0) for x in range(256)], dtype=np.int64)
_LOW = np.array([(x & -x).bit_length() - 1 if x else 0 for x in range(256)], dtype=np.int64)


def _u64(rec, o):
    return np.ascontiguousarray(rec[:, o:o + 8]).view("<u8")[:, 0]


def intake_numpy(rec, off, epoch, current_slot, domain, committees_per_slot, slots_per_epoch, bits_stride, parent, slot, roots):
    """intake_plain for n attestations of one length L, rec = uint8[n, L] (the wire reshaped), on the tree (parent, slot, roots)."""
    rec = np.asarray(rec, dtype=np.uint8)
    n, L = rec.shape
    off = np.asarray(off, dtype=np.int64)
    n_c, n_sig = off.shape[0] - 1, int(off[-1])
    status = np.zeros(n, dtype=np.int32)
    if L < FIXED:
        status[:] = 1
        return _numpy_votes(rec, status, None, None, off, n_c, n_sig, domain, None)
    status[np.ascontiguousarray(rec[:, :4]).view("<u4")[:, 0] != FIXED] = 1
    nb = L - FIXED
    if nb == 0:
        status[status == 0] = 2
        return _numpy_votes(rec, status, None, None, off, n_c, n_sig, domain, None)
    last = rec[:, L - 1]
    status[(status == 0) & (last == 0)] = 2
    top = _TOP[last]
    nbits = 8 * (nb - 1) + top
    status[(status == 0) & (nbits > 8 * bits_stride)] = 3
    live = status == 0
    payload = rec[:, FIXED:].copy()
    payload[:, -1] &= ((1 << top) - 1).astype(np.uint8)
    ones = _POP[payload].sum(axis=1, dtype=np.int64)
    status[live & (ones != 1)] = 4
    first_byte = np.argmax(payload != 0, axis=1)
    pos = 8 * first_byte + _LOW[payload[np.arange(n), first_byte]]
    s, idx, te = _u64(rec, 4), _u64(rec, 12), _u64(rec, 92)
    start = epoch * slots_per_epoch
    live = status == 0
    bad6 = (s < start) | (s >= start + slots_per_epoch) | (idx >= committees_per_slot)
    status[live & bad6] = 6
    live = status == 0
    c = np.where(live, (s - start) * committees_per_slot + idx, 0).astype(np.int64)
    status[live & (nbits != off[c + 1] - off[c])] = 5
    live = status == 0
    status[live & (te != epoch)] = 7
    live = status == 0
    status[live & (np.uint64(current_slot) < s + np.uint64(1))] = 8
    # checks 9-12 once per distinct data
    live = np.nonzero(status == 0)[0]
    data = np.ascontiguousarray(rec[live, 4:132]).view(np.dtype((np.void, 128)))[:, 0]
    uniq, inv = np.unique(data, return_inverse=True)
    roots = [bytes(r) for r in np.asarray(roots, dtype=np.uint8).reshape(-1, 32)]
    ids = {}
    for b, r in enumerate(roots):
        ids.setdefault(r, b)
    ustat, ublk = np.zeros(len(uniq), np.int32), np.zeros(len(uniq), np.int64)
    for k, u in enumerate(uniq):
        ustat[k], ublk[k] = _tree_check(bytes(u), ids, parent, slot, roots, start)
    status[live] = ustat[inv.reshape(-1)]
    # claims: the first passing attestation of each (committee, position); the later ones are duplicates
    keep = live[ustat[inv.reshape(-1)] == 0]
    key = c[keep] * (8 * bits_stride) + pos[keep]
    _, first = np.unique(key, return_index=True)
    dup = np.ones(keep.shape[0], dtype=bool)
    dup[first] = False
    status[keep[dup]] = 13
    win = keep[first]
    blk_of = np.zeros(n, np.int64)
    blk_of[live] = ublk[inv.reshape(-1)]
    return _numpy_votes(rec, status, c, pos, off, n_c, n_sig, domain, (win, blk_of))


def _tree_check(d: bytes, ids, parent, slot, roots, start):
    """checks 9-12 of one AttestationData: (status, head block id)"""
    head, target = d[16:48], d[96:128]
    if head not in ids:
        return 9, 0
    if target not in ids:
        return 10, 0
    h = ids[head]
    if int(slot[h]) > int.from_bytes(d[0:8], "little"):
        return 11, 0
    b = h
    while int(slot[b]) > start:
        if b == 0:
            return 12, 0
        b = int(parent[b])
    if roots[b] != target:
        return 12, 0
    return 0, h


def _numpy_votes(rec, status, c, pos, off, n_c, n_sig, domain, kept):
    """the vote form's arrays from the kept attestations (kept = (their indices, head block id per attestation) or None)"""
    vote = np.full(n_sig, NONE, dtype=np.uint32)
    sigs = np.zeros((n_sig, 96), dtype=np.uint8)
    counts = np.ones(n_c, dtype=np.int64)
    win, blk_of = kept if kept is not None else (np.zeros(0, np.int64), None)
    if win.size:
        wc, wp = c[win], pos[win]
        d = np.ascontiguousarray(rec[win, 4:132]).view(np.dtype((np.void, 128)))[:, 0]
        # groups = (committee, data); each group's smallest position orders the committee's votes
        _, g = np.unique(np.stack([wc.astype(np.int64), np.unique(d, return_inverse=True)[1].reshape(-1)], axis=1), axis=0, return_inverse=True)
        g = g.reshape(-1)
        n_g = int(g.max()) + 1
        gmin = np.full(n_g, np.iinfo(np.int64).max)
        np.minimum.at(gmin, g, wp)
        grep = np.zeros(n_g, np.int64)
        grep[g[wp == gmin[g]]] = win[wp == gmin[g]]
        gc = c[grep]
        order = np.lexsort((gmin, gc))
        kc = np.bincount(gc, minlength=n_c)
        counts = np.maximum(kc, 1)
        vote_off = np.concatenate([[0], np.cumsum(counts)])
        local = np.zeros(n_g, np.int64)
        starts = np.concatenate([[0], np.cumsum(kc)])
        local[order] = np.arange(n_g) - starts[gc[order]]
        gid = vote_off[gc] + local
        slots = off[wc] + wp
        vote[slots] = gid[g]
        sigs[slots] = rec[win, 132:228]
        rep_of_vote = np.full(int(vote_off[-1]), -1, np.int64)
        rep_of_vote[gid] = grep
    else:
        vote_off = np.concatenate([[0], np.cumsum(counts)])
        rep_of_vote = np.full(int(vote_off[-1]), -1, np.int64)
    rows = []
    for v in range(int(vote_off[-1])):
        a = int(rep_of_vote[v])
        if a < 0:
            rows.append((bytes(128), bytes(32), 0, 0, 0))
            continue
        db = rec[a, 4:132].tobytes()
        data = data_from_bytes(db)
        msg = compute_signing_root_from_object_root(hash_tree_root_attestation_data(data), domain)
        rows.append((db, msg, data.source.epoch, data.target.epoch, int(blk_of[a])))
    return _result(status, vote, vote_off.astype(np.int64), sigs, rows)


def encode(bits, data128: bytes, signature: bytes) -> bytes:
    from oracle.ssz import serialize_attestation
    return serialize_attestation(bits, data128, signature)


# ------------------------------------------------------------------------------------------ test epochs
def data128(slot, index, head, source_epoch, source_root, target_epoch, target_root) -> bytes:
    from oracle.ssz import serialize_attestation_data
    return serialize_attestation_data(slot, index, head, source_epoch, source_root, target_epoch, target_root)


def random_tree(rng, n_blocks, first_slot):
    """parent, slot, roots of a random tree whose slots increase strictly along every chain (what on_block builds)"""
    parent = np.zeros(n_blocks, dtype=np.uint32)
    slot = np.zeros(n_blocks, dtype=np.uint64)
    slot[0] = first_slot
    for b in range(1, n_blocks):
        parent[b] = rng.integers(0, b)
        slot[b] = slot[parent[b]] + rng.integers(1, 4)
    roots = rng.integers(0, 255, size=(n_blocks, 32), dtype=np.uint8)      # (never the all-0xff of block_store's outside root)
    roots[:, 0] = np.arange(n_blocks) % 251                                  # ... and distinct
    roots[:, 1] = np.arange(n_blocks) // 251
    return parent, slot, roots


def ancestor(parent, slot, b, at_slot):
    """get_ancestor by id; None when the walk leaves the tree"""
    while int(slot[b]) > at_slot:
        if b == 0:
            return None
        b = int(parent[b])
    return b


def random_epoch(rng, epoch, spe, cps, csize, tree, n_extra=0, corrupt=0.3, heads_per_committee=2):
    """The wires of one epoch: every member of every committee (all of size csize) attests once to one of a few heads of its committee;
    a share `corrupt` of them is broken in one way that keeps the record's length; n_extra duplicates of random earlier attestations
    are appended (some with other data)."""
    parent, slot, roots = tree
    start = epoch * spe
    wires, n_c = [], spe * cps
    src_root = bytes(roots[0])

    def good_data(c, pick):
        s = start + c // cps
        ok = [b for b in range(len(parent)) if int(slot[b]) <= s and ancestor(parent, slot, b, start) is not None]
        if not ok:
            ok = [0]
        h = ok[pick % len(ok)]
        t = ancestor(parent, slot, h, start)
        t = 0 if t is None else t
        return data128(s, c % cps, bytes(roots[h]), epoch - 1 if epoch else 0, src_root, epoch, bytes(roots[t]))

    for c in range(n_c):
        heads = [good_data(c, int(rng.integers(0, 1 << 30))) for _ in range(heads_per_committee)]
        for p in range(csize):
            d = bytearray(heads[int(rng.integers(0, len(heads)))])
            bits = [False] * csize
            bits[p] = True
            sig = rng.integers(0, 256, size=96, dtype=np.uint8).tobytes()
            kind = int(rng.integers(0, 12)) if rng.random() < corrupt else -1
            if kind == 0:
                bits[(p + 1) % csize] = True                                    # two bits (csize >= 2)
            elif kind == 1:
                bits[p] = False                                                 # no bit
            elif kind == 2:
                d[0:8] = (start + spe + 3).to_bytes(8, "little")                # foreign slot
            elif kind == 3:
                d[8:16] = (cps + 1).to_bytes(8, "little")                       # foreign index
            elif kind == 4:
                d[88:96] = (epoch + 1).to_bytes(8, "little")                    # target epoch
            elif kind == 5:
                d[16:48] = bytes([0xAB] * 32)                                   # unknown head
            elif kind == 6:
                d[96:128] = bytes([0xCD] * 32)                                  # unknown target
            elif kind == 7:
                d[16:48] = bytes(roots[int(np.argmax(slot))])                   # the newest block: usually newer than data.slot
            elif kind == 8:
                d[96:128] = bytes(roots[int(rng.integers(0, len(parent)))])    # a known block, usually not the ancestor
            w = bytearray(encode(bits, bytes(d), sig))
            if kind == 9:
                w[0] = 0                                                        # wrong offset
            elif kind == 10:
                w[-1] = 0                                                       # no delimiter
            elif kind == 11 and csize % 8 > 1:                                  # one bit shorter, the same bytes
                top = csize % 8 - 1
                w[-1] = (w[-1] & ((1 << top) - 1)) | (1 << top)
            wires.append(bytes(w))
    for _ in range(n_extra):
        w = bytearray(wires[int(rng.integers(0, len(wires)))])
        if rng.random() < 0.5:
            w[4 + 56] ^= 1                                                      # another source root: other data, same position
        wires.append(bytes(w))
    return wires


def ragged_layout(sizes):
    """the committee layout off (uint32[len(sizes) + 1]) of committees of the given sizes"""
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def ragged_epoch(rng, epoch, spe, cps, sizes, tree, distinct=2, absent=0.0, dup=0.0, corrupt=0.0):
    """The wires of one epoch whose committee c has sizes[c] members (len(sizes) == spe * cps).  Committee c's attesters sign
    distinct[c] (or `distinct`) different AttestationData, each used by at least one attester while min(that, attesters) allows; the
    data differ in their head or source root, so all of them pass the tree checks.  A share `absent` of the members does not attest.
    A share `corrupt` of the attestations fails one check: two bits (4), a Bitlist one bit longer (5), a foreign target epoch (7), an
    unknown head (9) or a known block that is not the target's ancestor as target (12).  The wires come in random order; then, for a
    share `dup` of the attestations, a second one for the same position is appended: with equal data, with other data, or after the
    earlier copy was made to fail (unknown target, 10), so that the appended one is the position's first passing attestation."""
    parent, slot, roots = tree
    start, n_c = epoch * spe, spe * cps
    assert len(sizes) == n_c
    distinct = [distinct] * n_c if np.isscalar(distinct) else list(distinct)
    src_root = bytes(roots[0])
    wires, meta = [], []
    for c in range(n_c):
        size, s = int(sizes[c]), start + c // cps
        ok = [b for b in range(len(parent)) if int(slot[b]) <= s and ancestor(parent, slot, b, start) is not None] or [0]
        present = np.nonzero(rng.random(size) >= absent)[0]
        k = max(1, min(int(distinct[c]), len(present)))
        group = rng.permutation(np.arange(len(present)) % k)
        data = []
        for g in range(k):
            h = ok[int(rng.integers(0, len(ok)))]
            t = ancestor(parent, slot, h, start)
            src = hashlib.sha256(b"ragged-source/%d/%d" % (c, g)).digest() if g else src_root
            data.append(data128(s, c % cps, bytes(roots[h]), epoch - 1 if epoch else 0, src, epoch, bytes(roots[0 if t is None else t])))
        for p, g in zip(present.tolist(), group.tolist()):
            meta.append((size, p, data[g]))
    sig = lambda: rng.integers(0, 256, size=96, dtype=np.uint8).tobytes()      # noqa: E731
    for size, p, d in meta:
        d, bits = bytearray(d), [j == p for j in range(size)]
        kind = int(rng.integers(0, 5)) if rng.random() < corrupt else -1
        if kind == 0 and size > 1:
            bits[(p + 1) % size] = True
        elif kind == 1:
            bits.append(False)
        elif kind == 2:
            d[88:96] = (epoch + 1).to_bytes(8, "little")
        elif kind == 3:
            d[16:48] = bytes([0xAB] * 32)
        elif kind == 4:
            d[96:128] = bytes(roots[int(np.argmax(slot))])
        wires.append(encode(bits, bytes(d), sig()))
    wires = [wires[i] for i in rng.permutation(len(wires))]
    for i in np.nonzero(rng.random(len(wires)) < dup)[0].tolist():
        w, kind = bytearray(wires[i]), int(rng.integers(0, 3))
        if kind == 1:
            w[4 + 56] ^= 1                                                      # other data, same position
        elif kind == 2:
            bad = bytearray(wires[i])
            bad[4 + 96:4 + 128] = bytes([0xCD] * 32)                            # the earlier copy fails (10)
            wires[i] = bytes(bad)
        w[132:228] = sig()
        wires.append(bytes(w))
    return wires
