"""CPU restatement of b2_block_attestations (csrc/blockatt.cuh): process_attestation (pos-evolution.md:722-754) for the attestations of a
run of blocks of one epoch, in the call's array form, block-atomic as on_block's state_transition (:1008-1009).  Sequential and literal:
the attestations one by one in (block, list) order, the blocks applied in order up to the first invalid one.  Also the wire helpers the
tests build their inputs with."""
import numpy as np

from intake_oracle import _decode, data128, encode  # noqa: F401  (data128 / encode: the tests' wire builders)
from oracle.spec import PARTICIPATION_FLAG_WEIGHTS, PROPOSER_WEIGHT, WEIGHT_DENOMINATOR, integer_squareroot
from oracle.ssz import compute_signing_root_from_object_root, htr_attestation_data

DENOMINATOR = (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT) * WEIGHT_DENOMINATOR // PROPOSER_WEIGHT     # :752, 448


def _u64(d, o):
    return int.from_bytes(d[o:o + 8], "little")


def signing_root(d: bytes, domain: bytes) -> bytes:
    root = htr_attestation_data(_u64(d, 0), _u64(d, 8), d[16:48], _u64(d, 48), d[56:88], _u64(d, 88), d[96:128])
    return compute_signing_root_from_object_root(root, domain)


def check(w: bytes, block_slot: int, e: int, members, off, cps_prev, cps_cur, chain_roots, justified80, domains64, spe, min_delay, bits_stride,
          verify):
    """(status, flag mask, target is e, selected members) of one attestation included at block_slot"""
    st, bits = _decode(w, 8 * bits_stride)
    if st:
        return st, 0, False, []
    d = w[4:132]
    slot, index, tgt = _u64(d, 0), _u64(d, 8), _u64(d, 88)
    cur = tgt == e
    cps = cps_cur if cur else cps_prev
    if not cur and (e == 0 or tgt != e - 1):
        return 4, 0, cur, []
    if tgt != slot // spe:
        return 5, 0, cur, []
    if not slot + min_delay <= block_slot <= slot + spe:
        return 6, 0, cur, []
    if index >= cps:
        return 7, 0, cur, []
    c = (cps_prev * spe if cur else 0) + (slot - tgt * spe) * cps + index
    o0, o1 = int(off[c]), int(off[c + 1])
    if not (o0 <= o1 <= len(members) and o1 - o0 <= 8 * bits_stride) or len(bits) != o1 - o0:
        return 8, 0, cur, []
    if d[48:88] != (justified80[40:80] if cur else justified80[0:40]):                       # is_matching_source (:733)
        return 9, 0, cur, []
    start = e * spe
    target = d[96:128] == bytes(chain_roots[spe if cur else 0])
    head = d[16:48] == bytes(chain_roots[slot + spe - start])
    delay = block_slot - slot
    mask = ((1 if delay <= integer_squareroot(spe) else 0) | (2 if target and delay <= spe else 0)
            | (4 if target and head and delay == min_delay else 0))
    selected = [int(members[o0 + j]) for j in range(len(bits)) if bits[j]]
    if not selected:
        return 10, mask, cur, []
    if not verify(sorted(set(selected)), signing_root(d, domains64[32:64] if cur else domains64[0:32]), w[132:228]):
        return 11, mask, cur, selected
    return 0, mask, cur, selected


def run(wire: bytes, woff, block_off, block_slot, members, off, cps_prev, cps_cur, chain_roots, justified80, domains64, spe, min_delay,
        bits_stride, eff, increment, per_increment, part_cur, part_prev, verify):
    """Everything the call returns, and the two participation tables after it.  chain_roots: 2 * spe roots, slot s at s + spe - start(e);
    verify(sorted indices, signing root, signature) -> bool is FastAggregateVerify."""
    n, n_blocks = len(woff) - 1, len(block_off) - 1
    e = int(block_slot[0]) // spe
    status, mask, numerator = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros(n, np.uint64)
    cur, sel = [False] * n, [[] for _ in range(n)]
    for b in range(n_blocks):
        for a in range(int(block_off[b]), int(block_off[b + 1])):
            if not int(woff[a]) <= int(woff[a + 1]) <= len(wire):
                status[a] = 1
                continue
            status[a], mask[a], cur[a], sel[a] = check(bytes(wire[int(woff[a]):int(woff[a + 1])]), int(block_slot[b]), e, members, off, cps_prev,
                                                       cps_cur, chain_roots, justified80, domains64, spe, min_delay, bits_stride, verify)
    block_status, block_first, block_reward = np.zeros(n_blocks, np.int32), np.full(n_blocks, 0xFFFFFFFF, np.uint32), np.zeros(n_blocks, np.uint64)
    for b in range(n_blocks):
        bad = [a for a in range(int(block_off[b]), int(block_off[b + 1])) if status[a]]
        if bad:
            block_status[b], block_first[b] = 1, bad[0] - int(block_off[b])
    invalid = [b for b in range(n_blocks) if block_status[b] == 1]
    n_applied = invalid[0] if invalid else n_blocks
    block_status[n_applied:][block_status[n_applied:] == 0] = 2
    tables = (list(part_cur), list(part_prev))
    for b in range(n_applied):
        for a in range(int(block_off[b]), int(block_off[b + 1])):
            table = tables[0 if cur[a] else 1]
            num = 0
            for v in sel[a]:                                                           # :745-749
                for f, weight in enumerate(PARTICIPATION_FLAG_WEIGHTS):
                    if (mask[a] >> f) & 1 and not (table[v] >> f) & 1:
                        table[v] |= 1 << f
                        num += (int(eff[v]) // increment) * per_increment * weight
            numerator[a] = num
            block_reward[b] += num // DENOMINATOR                                      # :752-754
    return dict(status=status, flag_mask=mask, numerator=numerator, block_status=block_status, block_first=block_first,
                block_reward=block_reward, n_applied=n_applied, part_cur=tables[0], part_prev=tables[1])


def layout(wires_per_block):
    """wire, woff, block_off of blocks given as lists of encodings"""
    flat = [w for blk in wires_per_block for w in blk]
    woff = np.concatenate([[0], np.cumsum([len(w) for w in flat])]).astype(np.uint32)
    block_off = np.concatenate([[0], np.cumsum([len(blk) for blk in wires_per_block])]).astype(np.uint32)
    return b"".join(flat), woff, block_off
