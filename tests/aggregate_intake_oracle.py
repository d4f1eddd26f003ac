"""Host oracle of the aggregated-attestation intake (include/b200pos.h, b2_aggregate_and_proof_intake): one target epoch of
SignedAggregateAndProof gossip messages checked item by item, in list order, as the status table of the header orders the upstream phase 0
beacon_aggregate_and_proof checks.

The validator helpers (is_aggregator, get_slot_signature's and get_aggregate_and_proof_signature's messages) are restated from upstream
phase 0; hash_tree_root(AggregateAndProof) is built from tests/ssz_oracle.py's merkleize / mix_in_length, independently of the product.
Signature verdicts come from the caller (`sig_ok`): known by construction (signed by the right key over the right message, or planted
corrupt), or computed with oracle.bls_sig on small cases."""
import hashlib
import types

import numpy as np

import ssz_oracle as S
from intake_oracle import _tree_check, encode as attestation_encode

NONE = 0xFFFFFFFF
OUTER, INNER = 100, 108
ATT = OUTER + INNER
BITLIST_LIMIT = 2048                    # MAX_VALIDATORS_PER_COMMITTEE
DOMAIN_BEACON_ATTESTER = bytes.fromhex("01000000")
DOMAIN_SELECTION_PROOF = bytes.fromhex("05000000")
DOMAIN_AGGREGATE_AND_PROOF = bytes.fromhex("06000000")


# ------------------------------------------------------------------------------------------ upstream phase 0 validator helpers
def is_aggregator(committee_len: int, selection_proof: bytes, target: int = 16) -> bool:
    modulo = max(1, committee_len // target)
    return int.from_bytes(hashlib.sha256(bytes(selection_proof)).digest()[0:8], "little") % modulo == 0


def signing_root(object_root: bytes, domain: bytes) -> bytes:
    """compute_signing_root: hash_tree_root(SigningData(object_root, domain))"""
    return S.merkleize([bytes(object_root), bytes(domain)])


def slot_signing_root(slot: int, domain: bytes) -> bytes:
    """the message of get_slot_signature: compute_signing_root(Slot(slot), selection-proof domain)"""
    return signing_root(S.uint_root(slot), domain)


def bitlist_root(bits, limit: int = BITLIST_LIMIT) -> bytes:
    packed = bytearray((len(bits) + 7) // 8)
    for i, b in enumerate(bits):
        if b:
            packed[i >> 3] |= 1 << (i & 7)
    return S.mix_in_length(S.merkleize(S.pack(bytes(packed)), limit=(limit + 255) // 256), len(bits))


def signature_root(sig: bytes) -> bytes:
    return S.merkleize(S.pack(bytes(sig)))


def data_root(d: bytes) -> bytes:
    cp = lambda o: S.merkleize([S.uint_root(int.from_bytes(d[o:o + 8], "little")), bytes(d[o + 8:o + 40])])      # noqa: E731
    return S.merkleize([S.uint_root(int.from_bytes(d[0:8], "little")), S.uint_root(int.from_bytes(d[8:16], "little")), bytes(d[16:48]), cp(48), cp(88)])


def attestation_root(bits, d: bytes, sig: bytes) -> bytes:
    return S.merkleize([bitlist_root(bits), data_root(d), signature_root(sig)])


def aggregate_and_proof_root(aggregator: int, bits, d: bytes, agg_sig: bytes, proof: bytes) -> bytes:
    return S.merkleize([S.uint_root(aggregator), attestation_root(bits, d, agg_sig), signature_root(proof)])


def aggregate_and_proof_signing_root(aggregator, bits, d, agg_sig, proof, domain) -> bytes:
    """the message of get_aggregate_and_proof_signature"""
    return signing_root(aggregate_and_proof_root(aggregator, bits, d, agg_sig, proof), domain)


def encode(aggregator: int, bits, d: bytes, agg_sig: bytes, proof: bytes, signature: bytes) -> bytes:
    """SSZ of SignedAggregateAndProof{AggregateAndProof{aggregator, Attestation{bits, d, agg_sig}, proof}, signature}"""
    return ((OUTER).to_bytes(4, "little") + bytes(signature) + int(aggregator).to_bytes(8, "little") + (INNER).to_bytes(4, "little") + bytes(proof)
            + attestation_encode(list(bits), bytes(d), bytes(agg_sig)))


def decode(w: bytes, max_bits: int):
    """(status 1-3 or 0, fields): fields = (aggregator, bits, data, aggregate signature, selection proof, signature)"""
    if len(w) < ATT + 228 or int.from_bytes(w[:4], "little") != OUTER or int.from_bytes(w[OUTER + 8:OUTER + 12], "little") != INNER:
        return 1, None
    a = w[ATT:]
    if int.from_bytes(a[:4], "little") != 228:
        return 1, None
    b = a[228:]
    if len(b) == 0 or b[-1] == 0:
        return 2, None
    n = 8 * (len(b) - 1) + b[-1].bit_length() - 1
    if n > max_bits:
        return 3, None
    bits = [bool((b[i >> 3] >> (i & 7)) & 1) for i in range(n)]
    return 0, (int.from_bytes(w[OUTER:OUTER + 8], "little"), bits, bytes(a[4:132]), bytes(a[132:228]), bytes(w[OUTER + 12:OUTER + 108]), bytes(w[4:100]))


def validate(wires, members, off, epoch, current_slot, domains96, committees_per_slot, slots_per_epoch, bits_stride, parent, slot, roots,
             sig_ok, target=16, propagation_range=32):
    """The statuses (0-20) and outputs of one call.  sig_ok(i) -> (selection proof valid, signature valid, aggregate valid) of item i,
    asked only for items that reach check 14.  The tree: parent ids, slots, roots of the device tree (block 0 its root)."""
    members, off = np.asarray(members, np.int64), np.asarray(off, np.int64)
    roots = [bytes(r) for r in np.asarray(roots, np.uint8).reshape(-1, 32)]
    ids = {}
    for b, r in enumerate(roots):
        ids.setdefault(r, b)
    dom_att = bytes(domains96[0:32])
    n, W = len(wires), 8 * bits_stride
    r = types.SimpleNamespace(status=np.zeros(n, np.int32), committee=np.full(n, NONE, np.uint32), data_id=np.full(n, NONE, np.uint32),
                              bits=np.zeros((n, bits_stride), np.uint8), sigs=np.zeros((n, 96), np.uint8), msgs=np.zeros((n, 32), np.uint8),
                              target_epoch=np.zeros(n, np.uint64), block_idx=np.full(n, NONE, np.uint32), members=np.zeros((n, W), np.uint32),
                              item_off=np.arange(n + 1, dtype=np.uint32) * W)
    first_data = {}
    accepted_bits, accepted_aggs = {}, set()      # the accepted items so far: bit lists per data, aggregators
    start = epoch * slots_per_epoch
    for i, w in enumerate(wires):
        st, f = decode(bytes(w), W)
        if st:
            r.status[i] = st
            continue
        agg, bits, d, agg_sig, proof, _ = f
        u = lambda o: int.from_bytes(d[o:o + 8], "little")      # noqa: E731
        s, index, tgt = u(0), u(8), u(88)
        first_data.setdefault(d, i)
        r.data_id[i] = first_data[d]
        row = bytearray(bits_stride)
        for j, b in enumerate(bits):
            if b:
                row[j >> 3] |= 1 << (j & 7)
        r.bits[i] = np.frombuffer(bytes(row), np.uint8)
        r.sigs[i] = np.frombuffer(agg_sig, np.uint8)
        r.msgs[i] = np.frombuffer(signing_root(data_root(d), dom_att), np.uint8)
        r.target_epoch[i] = tgt
        r.block_idx[i] = ids.get(d[16:48], NONE)
        se = s // slots_per_epoch
        if index >= committees_per_slot:
            st = 4
        elif not (s <= current_slot <= s + propagation_range):
            st = 5
        elif tgt != se:
            st = 6
        elif se != epoch:
            st = 7
        else:
            c = (s - start) * committees_per_slot + index
            com = members[off[c]:off[c + 1]].tolist()
            r.committee[i] = c
            r.members[i, :len(com)] = com
            if len(bits) != len(com):
                st = 8
            elif not any(bits):
                st = 9
            elif any(all(b <= ab for b, ab in zip(bits, a_b)) for a_b in accepted_bits.get(d, ())):
                st = 10
            elif agg in accepted_aggs:
                st = 11
            elif not is_aggregator(len(com), proof, target):
                st = 12
            elif agg not in com:
                st = 13
            else:
                ok_sel, ok_sig, ok_agg = sig_ok(i)
                if not ok_sel:
                    st = 14
                elif not ok_sig:
                    st = 15
                elif not ok_agg:
                    st = 16
                else:
                    t, _ = _tree_check(d, ids, parent, slot, roots, start)
                    st = 8 + t if t else 0
            if st == 0:
                accepted_bits.setdefault(d, []).append(bits)
                accepted_aggs.add(agg)
        r.status[i] = st
    return r
