"""CPU restatement of b2_block_attestations_electra (csrc/blockatt_electra.cuh): process_attestation for the Electra (EIP-7549) on-chain
Attestation with Deneb's (EIP-7045) inclusion window and flags (upstream consensus-specs, Deneb and Electra beacon-chain.md), for the
attestations of a run of blocks of one epoch, in the call's array form, block-atomic as on_block's state_transition.  Sequential and
literal: the attestations one by one in (block, list) order, each committee of an attestation by increasing index, the blocks applied in
order up to the first invalid one.  Also the Electra wire builders the tests use."""
import numpy as np

from block_attestations_oracle import DENOMINATOR, data128, signing_root  # noqa: F401  (data128: the tests' wire builder)
from oracle.spec import PARTICIPATION_FLAG_WEIGHTS, integer_squareroot


def fixed(M):
    """the fixed part: offset, AttestationData, signature, committee_bits (236 bytes on mainnet, 229 on minimal)"""
    return 4 + 128 + 96 + (M + 7) // 8


def bitvector(committee_bits) -> bytes:
    out = bytearray((len(committee_bits) + 7) // 8)
    for i, b in enumerate(committee_bits):
        if b:
            out[i >> 3] |= 1 << (i & 7)
    return bytes(out)


def bitlist(bits) -> bytes:
    out = bytearray(len(bits) // 8 + 1)
    for i, b in enumerate(bits):
        if b:
            out[i >> 3] |= 1 << (i & 7)
    out[len(bits) >> 3] |= 1 << (len(bits) & 7)
    return bytes(out)


def encode(bits, data: bytes, signature: bytes, committee_bits) -> bytes:
    """the Electra Attestation's SSZ encoding; committee_bits: M booleans"""
    assert len(data) == 128 and len(signature) == 96
    return fixed(len(committee_bits)).to_bytes(4, "little") + data + signature + bitvector(committee_bits) + bitlist(bits)


def committee_bits_of(indices, M):
    return [i in set(indices) for i in range(M)]


def _u64(d, o):
    return int.from_bytes(d[o:o + 8], "little")


def decode(w: bytes, M: int, limit: int):
    """(status 1-3 or 0, aggregation bits, committee bits)"""
    F = fixed(M)
    if len(w) < F or int.from_bytes(w[:4], "little") != F:
        return 1, None, None
    cb = w[228:F]
    if M % 8 and cb[-1] >> (M % 8):
        return 1, None, None                                   # a Bitvector with a padding bit set
    b = w[F:]
    if len(b) == 0 or b[-1] == 0:
        return 2, None, None
    n = 8 * (len(b) - 1) + b[-1].bit_length() - 1
    if n > limit:
        return 3, None, None
    return 0, [bool((b[i >> 3] >> (i & 7)) & 1) for i in range(n)], [bool((cb[i >> 3] >> (i & 7)) & 1) for i in range(M)]


def check(w: bytes, block_slot: int, e: int, members, off, cps_prev, cps_cur, chain_roots, justified80, domains64, spe, min_delay, M, max_vpc,
          verify, row_max=None):
    """(status, flag mask, target is e, attesting indices) of one attestation included at block_slot"""
    st, bits, cbits = decode(w, M, max_vpc * M)
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
    if not slot + min_delay <= block_slot:                                   # Deneb: no upper bound
        return 6, 0, cur, []
    if index != 0:
        return 7, 0, cur, []
    committee_offset, attesting = 0, set()
    for committee_index in [i for i, b in enumerate(cbits) if b]:           # get_committee_indices
        if committee_index >= cps:
            return 8, 0, cur, []
        c = (cps_prev * spe if cur else 0) + (slot - tgt * spe) * cps + committee_index
        o0, o1 = int(off[c]), int(off[c + 1])
        if not o0 <= o1 <= len(members) or (row_max is not None and committee_offset + o1 - o0 > row_max):
            return 10, 0, cur, []                                            # a malformed committee row
        committee = [int(v) for v in members[o0:o1]]
        if committee_offset + len(committee) > len(bits):
            return 10, 0, cur, []                                            # reading past the Bitlist's end
        committee_attesters = set(v for i, v in enumerate(committee) if bits[committee_offset + i])
        if not committee_attesters:
            return 9, 0, cur, []
        attesting |= committee_attesters
        committee_offset += len(committee)
    if len(bits) != committee_offset:
        return 10, 0, cur, []
    if d[48:88] != (justified80[40:80] if cur else justified80[0:40]):     # is_matching_source
        return 11, 0, cur, []
    start = e * spe
    target = d[96:128] == bytes(chain_roots[spe if cur else 0])
    head = d[16:48] == bytes(chain_roots[slot + spe - start])
    delay = block_slot - slot
    mask = (1 if delay <= integer_squareroot(spe) else 0) | (2 if target else 0) | (4 if target and head and delay == min_delay else 0)
    if not attesting:
        return 12, mask, cur, []
    if not verify(sorted(attesting), signing_root(d, domains64[32:64] if cur else domains64[0:32]), w[132:228]):
        return 13, mask, cur, sorted(attesting)
    return 0, mask, cur, sorted(attesting)


def run(wire: bytes, woff, block_off, block_slot, members, off, cps_prev, cps_cur, chain_roots, justified80, domains64, spe, min_delay, M,
        max_vpc, eff, increment, per_increment, part_cur, part_prev, verify):
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
                                                       cps_cur, chain_roots, justified80, domains64, spe, min_delay, M, max_vpc, verify)
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
            for v in sel[a]:
                for f, weight in enumerate(PARTICIPATION_FLAG_WEIGHTS):
                    if (mask[a] >> f) & 1 and not (table[v] >> f) & 1:
                        table[v] |= 1 << f
                        num += (int(eff[v]) // increment) * per_increment * weight
            numerator[a] = num
            block_reward[b] += num // DENOMINATOR
    return dict(status=status, flag_mask=mask, numerator=numerator, block_status=block_status, block_first=block_first,
                block_reward=block_reward, n_applied=n_applied, part_cur=tables[0], part_prev=tables[1])


def row_max(off, cps_prev, cps_cur, spe):
    """the largest member count of one slot's committees over e - 1 and e (what the host form computes; at least 1)"""
    off = np.asarray(off, np.int64)
    best = 1
    for s in range(2 * spe):
        cps = cps_prev if s < spe else cps_cur
        c = s * cps_prev if s < spe else cps_prev * spe + (s - spe) * cps_cur
        best = max(best, int(off[c + cps] - off[c]))
    return best
